"""VPQ and STQ of VIPSeg from per-frame joint label histograms: host side, numpy only.

A video's frames are described by two sorted id tables (``gt_ids``, ``pred_ids``: every id of the video's JSON entries,
plus 0 = VOID at index 0) and one int histogram per frame, ``hist[t, i, j]`` = pixels whose ground-truth id is
``gt_ids[i]`` and predicted id is ``pred_ids[j]``; the last row / column counts ids that are not in the table.  Every
number of the reference metrics is a regrouping of those cells:

* VPQ (deva/vps_metrics/eval_vpq_vipseg.py:106-257): a window's intersections are the sum of its frames' histograms,
  taken as the difference of two int64 prefix sums; its prediction areas are that sum's column sums.  The reference's
  ``np.unique`` over ``gt * 2^24 + pred`` lists pairs in ascending (gt id, pred id) order, which is the row-major order
  of the non-zero cells, so the per-category IoU sums accumulate in the reference's order and are equal bit for bit.
* STQ (eval_stq_vipseg.py:50-168, segmentation_and_tracking_quality.py): each table entry maps to one (semantic,
  instance) label per frame, so the confusion matrix, tube areas and intersections are sums of cells grouped by label,
  and the dicts are filled in the reference's order (ascending label within a frame, frames in order).
"""
import numpy as np

NFRAMES = (1, 2, 4, 6, 8, 10, 999)
OFFSET = 256 * 256 * 256
VOID = 0
# eval_stq_vipseg.py's constants
N_CLASSES = 124
IGNORE_LABEL = 255
BIT_SHIFT = 16
STQ_OFFSET = 2 ** 24
_EPSILON = 1e-15


def id_table(frames_json) -> np.ndarray:
    """Sorted int32 ids of every segment listed in a video's frame entries, with 0 (VOID) first."""
    ids = {0}
    for frame in frames_json:
        ids.update(int(el['id']) for el in frame['segments_info'])
    return np.array(sorted(ids), dtype=np.int32)


def frame_segments(segments_info):
    """The reference's per-frame segment dict: the first entry of an id is kept, duplicate entries add their area."""
    segms = {}
    for el in segments_info:
        if el['id'] in segms:
            segms[el['id']]['area'] += el['area']
        else:
            segms[el['id']] = dict(el)
    return segms


# ------------------------------------------------------------------------------------------------------------ VPQ
class PQStatCat:
    __slots__ = ('iou', 'tp', 'fp', 'fn')

    def __init__(self):
        self.iou, self.tp, self.fp, self.fn = 0.0, 0, 0, 0


class PQStat(dict):
    """category id -> PQStatCat; ``+=`` adds per category like the reference's ``PQStat.__iadd__``."""

    def __missing__(self, key):
        self[key] = v = PQStatCat()
        return v

    def __iadd__(self, other):
        for label, o in other.items():
            s = self[label]
            s.iou += o.iou
            s.tp += o.tp
            s.fp += o.fp
            s.fn += o.fn
        return self

    def pq_average(self, categories, isthing):
        pq, sq, rq, n = 0, 0, 0, 0
        per_class = {}
        for label, info in categories.items():
            if isthing is not None and isthing != (info['isthing'] == 1):
                continue
            s = self[label]
            iou, tp, fp, fn = s.iou, s.tp, s.fp, s.fn
            if tp + fp + fn == 0:
                per_class[label] = {'pq': 0.0, 'sq': 0.0, 'rq': 0.0, 'iou': 0.0, 'tp': 0, 'fp': 0, 'fn': 0}
                continue
            n += 1
            pq_class = iou / (tp + 0.5 * fp + 0.5 * fn)
            sq_class = iou / tp if tp != 0 else 0
            rq_class = tp / (tp + 0.5 * fp + 0.5 * fn)
            per_class[label] = {'pq': pq_class, 'sq': sq_class, 'rq': rq_class, 'iou': iou, 'tp': tp, 'fp': fp,
                                'fn': fn}
            pq += pq_class
            sq += sq_class
            rq += rq_class
        return {'pq': pq / n, 'sq': sq / n, 'rq': rq / n, 'n': n}, per_class


def check_prediction_frame(pan_pred_labels, pred_segms, categories):
    """The reference's prediction sanity checks of one frame (eval_vpq_vipseg.py:145-163), given the ascending ids
    present in the PNG; raises its KeyErrors.  The set receives the distinct ids in the order of the entries and loses
    them in the same order as the reference's, so the second error lists them in the same order."""
    pred_labels_set = set(el_id for el_id in pred_segms)
    for label in pan_pred_labels:
        if label not in pred_segms:
            if label == VOID:
                continue
            raise KeyError('Segment with ID {} is presented in PNG and not presented in JSON.'.format(label))
        pred_labels_set.remove(label)
        if pred_segms[label]['category_id'] not in categories:
            raise KeyError('Segment with ID {} has unknown category_id {}.'.format(
                label, pred_segms[label]['category_id']))
    if len(pred_labels_set) != 0:
        raise KeyError('The following segment IDs {} are presented in JSON and not presented in PNG.'.format(
            list(pred_labels_set)))


class VpqVideo:
    """One video's frames for VPQ: the checks run at construction (frame order, as the reference's first window size
    meets them); ``stat(nframes)`` is the video's PQStat for one window size."""

    def __init__(self, gt_js, pred_js, gt_ids, pred_ids, hist, categories, pred_png_labels=None):
        t_len = len(gt_js)
        assert hist.shape == (t_len, len(gt_ids) + 1, len(pred_ids) + 1), hist.shape
        self.categories = categories
        self.gt_ids, self.pred_ids = gt_ids, pred_ids
        self.g_index = {int(v): i for i, v in enumerate(gt_ids)}
        self.p_index = {int(v): j for j, v in enumerate(pred_ids)}
        self.gt_segms = [frame_segments(f['segments_info']) for f in gt_js]
        self.pred_segms = []
        cols = hist.sum(axis=1, dtype=np.int64)  # [T, P + 1] pixels per pred index
        for t, frame in enumerate(pred_js):
            segms = frame_segments(frame['segments_info'])
            present = np.nonzero(cols[t])[0]
            if cols[t, -1]:
                # an id that is in no JSON entry of the video: only the PNG knows which, so ask it (error path only)
                labels = pred_png_labels(t)
            else:
                labels = [int(pred_ids[j]) for j in present]
            check_prediction_frame(labels, segms, categories)
            for el_id, s in segms.items():
                s['area'] = cols[t, self.p_index[el_id]]
            self.pred_segms.append(segms)
        self.prefix = np.zeros((t_len + 1,) + hist.shape[1:], dtype=np.int64)
        np.cumsum(hist, axis=0, dtype=np.int64, out=self.prefix[1:])
        self.t_len = t_len

    def stat(self, nframes):
        stat = PQStat()
        for idx in range(0, max(self.t_len - nframes + 1, 1)):
            self._window(stat, idx, min(idx + nframes, self.t_len))
        return stat

    def _window(self, stat, a, b):
        vid_gt, vid_pred = {}, {}
        for t in range(a, b):
            for k, v in self.gt_segms[t].items():
                if k not in vid_gt:
                    vid_gt[k] = dict(v)
                else:
                    vid_gt[k]['area'] += v['area']
            for k, v in self.pred_segms[t].items():
                if k not in vid_pred:
                    vid_pred[k] = dict(v)
                else:
                    vid_pred[k]['area'] += v['area']
        m = self.prefix[b] - self.prefix[a]
        n_rows, n_cols = m.shape
        g_cat = np.full(n_rows, -1, np.int64)
        g_ok = np.zeros(n_rows, bool)  # in the window's JSON and not crowd
        g_area = np.zeros(n_rows, np.int64)
        for k, info in vid_gt.items():
            r = self.g_index[k]
            g_cat[r] = info['category_id']
            g_area[r] = info['area']
            g_ok[r] = info['iscrowd'] != 1
        p_cat = np.full(n_cols, -2, np.int64)
        p_area = np.zeros(n_cols, np.int64)
        for k, info in vid_pred.items():
            c = self.p_index[k]
            p_cat[c] = info['category_id']
            p_area[c] = info['area']
        rows, cols = np.nonzero(m)  # row-major: ascending (gt id, pred id)
        inter = m[rows, cols]
        cand = g_ok[rows] & (g_cat[rows] == p_cat[cols])
        rows, cols, inter = rows[cand], cols[cand], inter[cand]
        union = p_area[cols] + g_area[rows] - inter - m[0, cols]
        iou = inter / union
        gt_matched, pred_matched = set(), set()
        for r, c, v in zip(rows[iou > 0.5].tolist(), cols[iou > 0.5].tolist(), iou[iou > 0.5].tolist()):
            s = stat[int(g_cat[r])]
            s.tp += 1
            s.iou += v
            gt_matched.add(int(self.gt_ids[r]))
            pred_matched.add(int(self.pred_ids[c]))
        crowd = {}
        for gt_label, info in vid_gt.items():
            if gt_label in gt_matched:
                continue
            if info['iscrowd'] == 1:
                crowd[info['category_id']] = gt_label
                continue
            stat[info['category_id']].fn += 1
        for pred_label, info in vid_pred.items():
            if pred_label in pred_matched:
                continue
            c = self.p_index[pred_label]
            intersection = m[0, c]
            if info['category_id'] in crowd:
                intersection += m[self.g_index[crowd[info['category_id']]], c]
            if intersection / info['area'] > 0.5:
                continue
            stat[info['category_id']].fp += 1


def vpq_results(stat, categories):
    metrics = [('All', None), ('Things', True), ('Stuff', False)]
    results = {}
    for name, isthing in metrics:
        results[name], per_class = stat.pq_average(categories, isthing=isthing)
        if name == 'All':
            results['per_class'] = per_class
    return results


def vpq_text(results) -> str:
    """vpq-{n}.txt, byte for byte as eval_vpq_vipseg.vpq_compute writes it."""
    out = ['================================================\n',
           '{:10s}| {:>5s}  {:>5s}  {:>5s} {:>5s}'.format('', 'PQ', 'SQ', 'RQ', 'N\n'), '-' * (10 + 7 * 4) + '\n']
    for name in ('All', 'Things', 'Stuff'):
        r = results[name]
        out.append('{:10s}| {:5.1f}  {:5.1f}  {:5.1f} {:5d}\n'.format(name, 100 * r['pq'], 100 * r['sq'],
                                                                     100 * r['rq'], r['n']))
    out.append('{:4s}| {:>5s} {:>5s} {:>5s} {:>6s} {:>7s} {:>7s} {:>7s}\n'.format('IDX', 'PQ', 'SQ', 'RQ', 'IoU', 'TP',
                                                                                   'FP', 'FN'))
    for idx, r in results['per_class'].items():
        out.append('{:4d} | {:5.1f} {:5.1f} {:5.1f} {:6.1f} {:7d} {:7d} {:7d}\n'.format(
            idx, 100 * r['pq'], 100 * r['sq'], 100 * r['rq'], r['iou'], r['tp'], r['fp'], r['fn']))
    return ''.join(out)


def vpq_simple_text(vpqs) -> str:
    """vpq-simple.txt from [(all, thing, stuff)] per window size."""
    return ''.join(f'{a:.1f}/{t:.1f}/{s:.1f},' for a, t, s in vpqs)


# ------------------------------------------------------------------------------------------------------------ STQ
def instance_numbers(frames_json):
    """id -> instance number, in order of first appearance over the video's entries."""
    numbers = {}
    for frame in frames_json:
        for el in frame['segments_info']:
            if el['id'] not in numbers:
                numbers[el['id']] = len(numbers)
    return numbers


def _labels(table, segments_info, numbers):
    """(semantic << 16) + instance per table entry (+ the not-in-table bucket) for one frame: ids absent from the
    frame's entries are 255 / 255; the last entry of an id wins."""
    sem = np.full(len(table) + 1, IGNORE_LABEL, np.int64)
    ins = np.full(len(table) + 1, 255, np.int64)
    index = {int(v): i for i, v in enumerate(table)}
    for el in segments_info:
        i = index[el['id']]
        sem[i] = el['category_id']
        ins[i] = numbers[el['id']]
    return ((sem << BIT_SHIFT) + ins).astype(np.int32).astype(np.int64)


def _group(values, counts):
    """Ascending distinct values and the summed int64 counts (np.unique's order)."""
    u, inv = np.unique(values, return_inverse=True)
    s = np.zeros(len(u), np.int64)
    np.add.at(s, inv, counts)
    return u, s


def _update(stat_dict, values, counts):
    for k, v in zip(*_group(values, counts)):
        if k in stat_dict:
            stat_dict[k] += v
        else:
            stat_dict[k] = v


class STQuality:
    """The reference's STQuality (num_classes 124, ignore 255 -> class 124, 16-bit label shift, offset 2^24) fed with
    histogram cells instead of pixels."""

    def __init__(self, things_list):
        self.things = np.array(sorted(set(things_list)), np.int64)
        self.size = N_CLASSES + 1
        self.include = np.arange(N_CLASSES)
        self.confusion, self.predictions, self.ground_truth, self.intersections, self.length = {}, {}, {}, {}, {}

    def update_video(self, seq_id, gt_js, pred_js, gt_ids, pred_ids, hist):
        gt_numbers, pred_numbers = instance_numbers(gt_js), instance_numbers(pred_js)
        for t in range(len(gt_js)):
            y_true = _labels(gt_ids, gt_js[t]['segments_info'], gt_numbers)
            y_pred = _labels(pred_ids, pred_js[t]['segments_info'], pred_numbers)
            self.update_cells(seq_id, y_true, y_pred, hist[t])

    def update_cells(self, seq_id, y_true, y_pred, hist):
        rows, cols = np.nonzero(hist)
        counts = hist[rows, cols].astype(np.int64)
        yt, yp = y_true[rows], y_pred[cols]
        sem_t, sem_p = yt >> BIT_SHIFT, yp >> BIT_SHIFT
        sem_t = np.where(sem_t != IGNORE_LABEL, sem_t, N_CLASSES)
        sem_p = np.where(sem_p != IGNORE_LABEL, sem_p, N_CLASSES)
        if seq_id not in self.confusion:
            self.confusion[seq_id] = np.zeros((self.size, self.size), np.int64)
            self.predictions[seq_id], self.ground_truth[seq_id], self.intersections[seq_id] = {}, {}, {}
            self.length[seq_id] = 0
        np.add.at(self.confusion[seq_id], (sem_t, sem_p), counts)
        self.length[seq_id] += 1
        label_mask = np.isin(sem_t, self.things)
        prediction_mask = np.isin(sem_p, self.things)
        is_crowd = ((yt & 0xFFFF) == 0) & label_mask
        label_mask &= ~is_crowd
        prediction_mask &= ~is_crowd
        _update(self.predictions[seq_id], yp[prediction_mask], counts[prediction_mask])
        _update(self.ground_truth[seq_id], yt[label_mask], counts[label_mask])
        both = label_mask & prediction_mask
        _update(self.intersections[seq_id], yt[both] * STQ_OFFSET + yp[both], counts[both])

    def result(self):
        n_seq = len(self.ground_truth)
        num_tubes, aq_per_seq, iou_per_seq, id_per_seq = [0] * n_seq, [0] * n_seq, [0] * n_seq, [''] * n_seq
        for index, seq_id in enumerate(self.ground_truth):
            outer_sum = 0.0
            predictions = self.predictions[seq_id]
            intersections = self.intersections[seq_id]
            ground_truth = self.ground_truth[seq_id]
            num_tubes[index] = len(ground_truth)
            id_per_seq[index] = seq_id
            # the reference's double loop visits, per ground-truth tube, the predictions in insertion order and keeps
            # those that intersect it; the same pairs in the same order, without the empty ones
            pred_order = {k: i for i, k in enumerate(predictions)}
            by_gt = {}
            for key in intersections:
                gt_id, pr_id = divmod(int(key), STQ_OFFSET)
                by_gt.setdefault(gt_id, []).append(pr_id)
            for gt_id, gt_size in ground_truth.items():
                inner_sum = 0.0
                for pr_id in sorted(by_gt.get(int(gt_id), ()), key=lambda p: pred_order[p]):
                    pr_size = predictions[pr_id]
                    tpa = intersections[STQ_OFFSET * gt_id + pr_id]
                    fpa = pr_size - tpa
                    fna = gt_size - tpa
                    inner_sum += tpa * (tpa / (tpa + fpa + fna))
                outer_sum += 1.0 / gt_size * inner_sum
            aq_per_seq[index] = outer_sum
        aq_mean = np.sum(aq_per_seq) / np.maximum(np.sum(num_tubes), _EPSILON)
        aq_per_seq = aq_per_seq / np.maximum(num_tubes, _EPSILON)
        total = np.zeros((self.size, self.size), np.int64)
        for index, confusion in enumerate(self.confusion.values()):
            removal = np.zeros_like(confusion)
            removal[self.include, :] = 1.0
            confusion = confusion * removal
            total += confusion
            inter = confusion.diagonal()
            unions = inter + (confusion.sum(axis=0) - inter) + (confusion.sum(axis=1) - inter)
            ious = inter.astype(np.double) / np.maximum(unions, 1e-15).astype(np.double)
            iou_per_seq[index] = np.sum(ious) / np.count_nonzero(unions)
        inter = total.diagonal()
        unions = inter + (total.sum(axis=0) - inter) + (total.sum(axis=1) - inter)
        ious = inter.astype(np.double) / np.maximum(unions, _EPSILON).astype(np.double)
        iou_mean = np.sum(ious) / np.count_nonzero(unions)
        return {'STQ': np.sqrt(aq_mean * iou_mean), 'AQ': aq_mean, 'IoU': float(iou_mean),
                'STQ_per_seq': np.sqrt(aq_per_seq * iou_per_seq), 'AQ_per_seq': aq_per_seq, 'IoU_per_seq': iou_per_seq,
                'ID_per_seq': id_per_seq, 'Length_per_seq': list(self.length.values())}


def stq_text(result) -> str:
    return f'{result["STQ"]*100:.1f},{result["AQ"]*100:.1f},{result["IoU"]*100:.1f}\n'


def thing_list(categories_list):
    return [c['id'] for c in categories_list if c['isthing']]


# ------------------------------------------------------------------------------------------------- stuff merging
class IDPostprocessor:
    """The reference's id rule (deva/utils/pano_utils.py:IDPostprocessor), drawing from the global np.random alike."""

    def __init__(self):
        self.all_id = []
        self.thing_obj_to_id = {}
        self.stuff_to_id = {}

    def _find_new_id(self, default_id):
        id = default_id
        while True:
            if id not in self.all_id:
                return id
            id = np.random.randint(256, 256 ** 3)

    def convert(self, obj, category_id, isthing):
        if isthing:
            if (obj, category_id) in self.thing_obj_to_id:
                return self.thing_obj_to_id[(obj, category_id)]
            id = self._find_new_id(obj)
            self.thing_obj_to_id[(obj, category_id)] = id
        else:
            if category_id in self.stuff_to_id:
                return self.stuff_to_id[category_id]
            id = self._find_new_id(obj)
            self.stuff_to_id[category_id] = id
        self.all_id.append(id)
        return id


def merge_plan(vid_ann, cat_to_isthing):
    """Host half of stuff merging for one video: the id rewrite of every frame and its thing entries.
    -> (pred id table, [(slot int32 [len(table) + 1], out_ids int32 [n_out], thing segments)], converter)."""
    table = id_table(vid_ann['annotations'])
    index = {int(v): i for i, v in enumerate(table)}
    converter = IDPostprocessor()
    frames = []
    for ann in vid_ann['annotations']:
        new = {}
        things = []
        for segment in ann['segments_info']:
            category_id = segment['category_id']
            isthing = cat_to_isthing[category_id]
            new_id = converter.convert(segment['id'], category_id, isthing)
            new[segment['id']] = new_id  # a later entry of the same id repaints its pixels
            if isthing:
                things.append({'id': new_id, 'category_id': category_id, 'isthing': 1})
        out_ids = [0] + sorted(set(v for v in new.values() if v != 0))
        slot_of = {v: s for s, v in enumerate(out_ids)}
        slot = np.zeros(len(table) + 1, np.int32)
        for k, v in new.items():
            slot[index[int(k)]] = slot_of[v]
        frames.append((slot, np.array(out_ids, np.int32), things, dict(converter.stuff_to_id)))
    return table, frames, converter


def merged_segments(things, stuff_to_id, out_ids, counts, cat_to_isthing):
    """A frame's output segments_info: things in entry order, then merged stuff with pixels, in stuff_to_id order."""
    area = {int(v): int(c) for v, c in zip(out_ids, counts)}
    out = list(things)
    for cat, new_id in stuff_to_id.items():
        assert not cat_to_isthing[cat]
        if area.get(new_id, 0) > 0:
            out.append({'id': new_id, 'category_id': cat, 'isthing': 0})
    return out
