"""Multi-GPU plumbing: channel-instance sharding (no data-path collective) and two optional exchanges.

Every metering instance is self-contained (SURVEY.md §8e), so N GPUs simply own contiguous instance ranges:
rank r of W processes instances  [r*n/W, (r+1)*n/W).  The only cross-instance quantity is the whole-mix gated
loudness: the int32 sum of all instances' hist_M / hist_S (+ counts), reduced per GPU by
b200m_ebu_mix_reduce and across GPUs by ONE all-reduce of B200M_MIX_WORDS int32 (NCCL on GPUs, gloo in CPU
tests); integer sums are order independent, hence bit-exact for any GPU count.  Album loudness works the same way with
one row per album (b200m_ebu_group_reduce): the clips of one album may sit on different GPUs.
The second exchange is album DR (b200m_dr14_group_reduce): each album's int32 row of summed window histograms and counts is
all-reduced the same way, but its window peaks cannot be summed (an album's second-highest window peak is the second largest over
all its tracks), so every rank's [G, nch, 3] peaks are all-gathered and b200m_dr14_group_finish merges the W parts by value.
Album spectra need no exchange of their own: gather_results collects each rank's per-clip sums, counts and peak_db of
programme_spectrum in clip order, and spectrum_albums pools them on the host exactly as it pools the rows of one bank.
Album correlation distributions likewise: gather_results collects each rank's per-clip hist and sums of programme_correlation,
and correlation_albums pools them on the host.
Album needle distributions too: gather_results collects each rank's per-clip hist and stats of programme_needle, and needle_albums
pools them on the host; every album value is an integer sum or a maximum, so any split of the clips gives the same result.
Album true-peak and K-meter distributions the same way: needle_albums pools each rank's per-clip tp_hist / tp_stats and km_hist /
km_stats of programme_truepeak.
Album stereo images too (gather_results + stereo_albums, no exchange): stereo_albums pools each rank's per-clip sums, analyses and
skipped of programme_stereo on the host.
"""
MIX_WORDS = 1508
DR14_HISTBINS = 8000


def shard_range(n_total, rank, world):
    """contiguous, balanced partition: returns (first, count) of the instances owned by `rank`."""
    if not (0 <= rank < world) or n_total < 0:
        raise ValueError("bad rank/world/n_total")
    lo = n_total * rank // world
    hi = n_total * (rank + 1) // world
    return lo, hi - lo


def shard_rows(n_total, nchan, rank, world):
    """row range of a planar [n_total*nchan, nfram] batch owned by `rank`."""
    lo, cnt = shard_range(n_total, rank, world)
    return lo * nchan, cnt * nchan


def allreduce_mix(mix, group=None):
    """sum the per-rank whole-mix histogram vector (int32[MIX_WORDS]), or the album rows of Ebu_r128_proc.group_reduce
    (int32[G, MIX_WORDS], the same G on every rank), over all ranks, in place."""
    import torch
    import torch.distributed as dist
    if mix.dtype != torch.int32 or not (mix.numel() == MIX_WORDS or (mix.dim() == 2 and mix.shape[1] == MIX_WORDS)):
        raise ValueError("mix must be int32[%d] or int32[G, %d]" % (MIX_WORDS, MIX_WORDS))
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(mix, op=dist.ReduceOp.SUM, group=group)
    return mix


def allreduce_dr14_groups(rows, peaks, group=None):
    """album DR across ranks: sum the rows of DR14.group_reduce (int32[G, nch * 8000 + 2], the same G on every rank) in place, and
    all-gather its peaks (float32[G, nch, 3]).  Returns the [W, G, nch, 3] stack of every rank's peaks in rank order (W = 1 without
    a process group), which DR14.group_finish takes with the summed rows."""
    import torch
    import torch.distributed as dist
    if rows.dtype != torch.int32 or rows.dim() != 2:
        raise ValueError("rows must be int32[G, nch * %d + 2]" % DR14_HISTBINS)
    g, words = rows.shape
    if peaks.dtype != torch.float32 or peaks.dim() != 3 or peaks.shape[0] != g or peaks.shape[2] != 3 \
            or words != peaks.shape[1] * DR14_HISTBINS + 2:
        raise ValueError("peaks must be float32[G, nch, 3] matching rows int32[G, nch * %d + 2]" % DR14_HISTBINS)
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(rows, op=dist.ReduceOp.SUM, group=group)
        p = peaks.contiguous()
        parts = [torch.empty_like(p) for _ in range(dist.get_world_size(group))]
        dist.all_gather(parts, p, group=group)
        return torch.stack(parts)
    return peaks.unsqueeze(0).contiguous()


def gather_results(local, group=None):
    """concatenate per-rank result arrays (numpy structured or plain) on every rank, in rank order."""
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return [local]
    out = [None] * dist.get_world_size(group)
    dist.all_gather_object(out, local, group=group)
    return out
