"""The data set feed's batch order (net.dataset_schedule, host/data.{h,cc} DataSchedule) against a restatement of the
reference's DataHandler (src/datahandler.cc:124-315) written here from the source, rule for rule.  Host logic only."""
import itertools

import pytest

from convnet_b200 import net

M64 = (1 << 64) - 1


class SplitMix:
    """host/data.cc SplitMix64, and the shuffle DataSchedule documents: j = next % (i + 1) for i = n-1 .. 1"""

    def __init__(self, state):
        self.s = state & M64

    def next(self):
        self.s = (self.s + 0x9E3779B97F4A7C15) & M64
        z = self.s
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
        return z ^ (z >> 31)

    def shuffle(self, v):
        for i in range(len(v), 1, -1):
            j = self.next() % i
            v[i - 1], v[j] = v[j], v[i - 1]


class RefDataHandler:
    """datahandler.cc's DataHandler without the data: what each GetBatch loads, slices and shuffles"""

    def __init__(self, c, dataset_size, seed):
        self.c, self.dataset_size = c, dataset_size
        self.cpu = SplitMix(seed * 0x9E3779B97F4A7C15 + 0x632BE59BD9B4E019)
        self.gpu = SplitMix(seed * 0x9E3779B97F4A7C15 + 0x8CB92BA72F3D8DD7)
        self.chunk_size, self.fits_on_gpu = c["chunk_size"], False
        if self.chunk_size <= 0 or self.chunk_size > dataset_size:
            self.chunk_size, self.fits_on_gpu = dataset_size, True
        self.nothing_on_gpu, self.random_indices_ind, self.preload = True, 0, None
        self.rand_perm_indices = list(range(self.chunk_size))                       # SetupShuffler
        if c["randomize_cpu"]:
            self.random_indices = list(range(dataset_size))
            self.cpu.shuffle(self.random_indices)
        self.seek(0)

    def seek(self, row):
        self.preload = None                                                         # Sync -> WaitForPreload
        self.start, self.reuse_counter, self.multiplicity_counter, self.restart = row, 0, 0, True
        self.row = row                                                              # DataIterator::Seek

    def disk_access(self):
        c, rows = self.c, []
        if c["randomize_cpu"]:
            racs = c["random_access_chunk_size"]
            num_rand = (self.chunk_size + racs - 1) // racs
            if self.random_indices_ind + num_rand > self.dataset_size:
                self.cpu.shuffle(self.random_indices)
                self.random_indices_ind = 0
            random_rows = self.random_indices[self.random_indices_ind:self.random_indices_ind + num_rand]
            self.random_indices_ind += num_rand
            for row in random_rows:                                                 # LoadChunk(it, mat, random_rows)
                end = (row + racs) % self.dataset_size
                if end < row:
                    rows += list(range(row, self.dataset_size)) + list(range(0, end))
                else:
                    rows += list(range(row, end))
        else:
            for _ in range(self.chunk_size):                                        # LoadChunk(it, mat): GetNext
                rows.append(self.row)
                self.row = (self.row + 1) % self.dataset_size
        return rows

    def get_batch(self):
        c, loaded = self.c, None
        end = self.start + c["batch_size"]
        if end > self.chunk_size or self.restart:
            if self.reuse_counter < c["max_reuse_count"] and not self.restart:
                self.reuse_counter += 1
            elif self.nothing_on_gpu or not self.fits_on_gpu:
                if self.restart and c["pipeline_loads"]:
                    self.preload = self.disk_access()                               # StartPreload
                self.nothing_on_gpu, self.reuse_counter = False, 0
                if c["pipeline_loads"]:                                             # PipelinedDiskAccess
                    loaded, self.preload = self.preload, None
                else:
                    loaded = self.disk_access()
                if c["pipeline_loads"]:
                    self.preload = self.disk_access()
            self.restart = False
            if c["randomize_gpu"]:
                self.gpu.shuffle(self.rand_perm_indices)                            # ShuffleIndices
            self.start, end = 0, c["batch_size"]
        out = (loaded, self.start, self.multiplicity_counter, list(self.rand_perm_indices))
        self.multiplicity_counter += 1
        if self.multiplicity_counter == c["multiplicity"]:
            self.multiplicity_counter, self.start = 0, end
        return out


def ref_schedule(config, dataset_size, steps, seed, seeks=None):
    c = dict(net.DatasetOrder.DEFAULTS, chunk_size=0, max_reuse_count=0, pipeline_loads=0, randomize_cpu=0, randomize_gpu=0)
    c.update(config)
    h, out = RefDataHandler(c, dataset_size, seed), []
    for k in range(steps):
        if seeks and k in seeks:
            h.seek(seeks[k])
        out.append(h.get_batch())
    return out


GRID = list(itertools.product((0, 1), (0, 1), (0, 1), (0, 2), (1, 10), ("fits", "3.5 chunks"), (1, 4)))


@pytest.mark.parametrize("pipeline,rcpu,rgpu,reuse,mult,size,racs", GRID)
def test_schedule_matches_reference_rules(pipeline, rcpu, rgpu, reuse, mult, size, racs):
    chunk, dataset = (0, 24) if size == "fits" else (8, 28)
    config = dict(batch_size=3, chunk_size=chunk, max_reuse_count=reuse, pipeline_loads=pipeline, randomize_cpu=rcpu,
                  randomize_gpu=rgpu, random_access_chunk_size=racs, multiplicity=mult)
    steps, seeks = 90, {41: 5, 63: 23}
    got = net.dataset_schedule(config, dataset, steps, seed=7, seeks=seeks)
    assert got == ref_schedule(config, dataset, steps, 7, seeks)
    chunk_size = chunk or dataset
    assert got[0][0] is not None                                # the first batch loads a chunk
    for rows, start, mid, perm in got:
        assert sorted(perm) == list(range(chunk_size))          # every pass reads a permutation of its chunk
        assert 0 <= start and start + 3 <= chunk_size and 0 <= mid < mult
        assert rows is None or (len(rows) == chunk_size and all(0 <= r < dataset for r in rows))
        if rows is not None and not rcpu:                       # consecutive rows, wrapping at the end of the data set
            assert rows == [(rows[0] + k) % dataset for k in range(chunk_size)]


def test_schedule_with_every_flag_off_is_the_plain_start_sequence():
    # what callers of DataIterator did by hand: start = 0, b, 2b, ... while a batch fits, then the next chunk of rows
    got = net.dataset_schedule(dict(batch_size=3, chunk_size=8), 28, 12)
    starts = [s for _, s, _, _ in got]
    assert starts == [0, 3, 0, 3, 0, 3, 0, 3, 0, 3, 0, 3]
    assert [r for r, _, _, _ in got][::2] == [[(8 * k + j) % 28 for j in range(8)] for k in range(6)]
    assert all(r is None for r, _, _, _ in got[1::2])
    assert all(m == 0 and p == list(range(8)) for _, _, m, p in got)
    fits = net.dataset_schedule(dict(batch_size=4), 12, 7)
    assert [s for _, s, _, _ in fits] == [0, 4, 8, 0, 4, 8, 0] and fits[0][0] == list(range(12))
    assert all(r is None for r, _, _, _ in fits[1:])           # a data set that fits is loaded once


def test_multiplicity_and_reuse():
    got = net.dataset_schedule(dict(batch_size=2, chunk_size=4, multiplicity=3, max_reuse_count=1), 8, 14)
    assert [(s, m) for _, s, m, _ in got] == [(0, 0), (0, 1), (0, 2), (2, 0), (2, 1), (2, 2)] * 2 + [(0, 0), (0, 1)]
    loads = [r for r, _, _, _ in got]
    assert loads[0] == [0, 1, 2, 3] and loads[12] == [4, 5, 6, 7]
    assert all(r is None for k, r in enumerate(loads) if k not in (0, 12))   # the chunk is reused once before the next


def test_pipelining_keeps_the_order_without_seek():
    base = dict(batch_size=3, chunk_size=8, randomize_cpu=1, randomize_gpu=1, random_access_chunk_size=4, max_reuse_count=1)
    assert (net.dataset_schedule(dict(base, pipeline_loads=1), 28, 60, seed=3) ==
            net.dataset_schedule(base, 28, 60, seed=3))


def test_refused_configurations():
    with pytest.raises(ValueError, match="does not divide the chunk"):
        net.dataset_schedule(dict(batch_size=2, chunk_size=8, randomize_cpu=1, random_access_chunk_size=3), 30, 1)
    # without randomize_cpu the field is not read, as in the reference
    net.dataset_schedule(dict(batch_size=2, chunk_size=8, random_access_chunk_size=3), 30, 1)
    with pytest.raises(ValueError, match="larger than the chunk"):
        net.dataset_schedule(dict(batch_size=9, chunk_size=8), 30, 1)
    with pytest.raises(ValueError, match="outside the data set"):
        net.dataset_schedule(dict(batch_size=2), 30, 2, seeks={1: 30})
    with pytest.raises(KeyError):
        net.dataset_schedule(dict(batch_size=2, shuffle=1), 30, 1)


MODEL = """name: "dsnet"
seed: 1
layer { name: "input" num_channels: 3 image_size_y: 12 image_size_x: 12 }
layer { name: "output" num_channels: 10 activation: SOFTMAX }
edge { source: "input" dest: "output" edge_type: FC }
train_dataset {
  batch_size: 16 chunk_size: 64 max_reuse_count: 2 pipeline_loads: true randomize_gpu: true multiplicity: 3
  data_config { file_pattern: "labels.h5" layer_name: "output" }
  data_config { file_pattern: "images.h5" layer_name: "input" can_translate: true can_flip: true
                gpu_image_size_y: 12 gpu_image_size_x: 12 }
}
"""


def test_model_dataset_reads_the_dataset_config(tmp_path):
    p = tmp_path / "ds.pbtxt"
    p.write_text(MODEL)
    d = net.model_dataset(str(p))
    assert d == dict(batch_size=16, chunk_size=64, max_reuse_count=2, pipeline_loads=True, randomize_cpu=False,
                     randomize_gpu=True, random_access_chunk_size=1, multiplicity=3, translate=True, flip=True,
                     gpu_image_size_y=12, gpu_image_size_x=12)
    assert net.model_dataset(str(p), "valid_dataset") is None
    assert "train_dataset" not in net.model_text(str(p))       # model_text writes the net, not its data
    assert net.model_dataset("lenet") is None
