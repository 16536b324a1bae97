// lv2_hub.cuh — host-side plumbing shared by the LV2 façade plugins (no device code): pinned staging of a cycle's input,
// the urid:map lookup, the audio forward, and the slot hub of batched mode.
#pragma once
#include <stdlib.h>
#include <string.h>
#include <mutex>
#include <vector>
#include "common.cuh"
#include "lv2_abi.cuh"

namespace b200m {

// Pinned [rows][cap] planar staging for *_process_host / *_run_host.  All-zero is the empty state (lv2_gon.cu callocs its
// plugin).  reserve() at instantiate sizes it for the largest cycle, so that run() never allocates; fill() allocates only
// when that failed.
struct PinnedStage {
    float* data = nullptr; size_t cap = 0;                    // cap: frames per row = the stride for *_process_host

    void reserve (uint32_t rows)
    {
        if (b200m_host_alloc ((void**)&data, (size_t)rows * B200M_MAX_BLOCK * sizeof (float)) == 0) cap = B200M_MAX_BLOCK;
    }
    // rows r < rows take n frames of in[r]; a null in[r] stages silence.  false: no staging memory.
    bool fill (const float* const* in, uint32_t rows, uint32_t n)
    {
        if (n > cap) {
            release ();
            const size_t c = n < 1024 ? 1024 : B200M_MAX_BLOCK;
            if (b200m_host_alloc ((void**)&data, (size_t)rows * c * sizeof (float))) { data = nullptr; return false; }
            cap = c;
        }
        for (uint32_t r = 0; r < rows; ++r) {
            if (in[r]) memcpy (data + r * cap, in[r], n * sizeof (float));
            else memset (data + r * cap, 0, n * sizeof (float));
        }
        return true;
    }
    void release ()
    {
        if (data) b200m_host_free (data);
        data = nullptr; cap = 0;
    }
};

inline LV2_URID_Map* find_urid_map (const LV2_Feature* const* features)
{
    for (int i = 0; features && features[i]; ++i)
        if (!strcmp (features[i]->URI, B200M_LV2_URID_MAP)) return (LV2_URID_Map*)features[i]->data;
    return nullptr;
}

// the in -> out copy every run() makes; in-place ports and unconnected ones are left alone
inline void forward_audio (float* const* in, float* const* out, uint32_t chn, uint32_t n)
{
    for (uint32_t c = 0; c < chn; ++c) if (in[c] && out[c] && in[c] != out[c]) memcpy (out[c], in[c], sizeof (float) * n);
}

// ---- batched mode (opt-in: B200M_LV2_BATCH=<slots>) ---------------------------------------------------------------------
// By default every façade instance is a synchronous bank of one: exact, but one upload / launch / download round trip per
// instance and cycle.  With B200M_LV2_BATCH=N the instances with one HubKey share ONE bank of N slots: run() copies its input
// into its rows of a pinned staging block and publishes the results of the PREVIOUS cycle (one declared cycle of latency on
// every reading; the audio pass-through is not delayed); the instance whose run() completes the cycle (every member has
// submitted) launches the bank asynchronously.
// Host contract: every instance runs once per cycle with the same n_samples.  When it is broken (an instance submits twice,
// or n_samples changes) the open cycle is launched as it is, and the rows of the members that did not submit are zeroed
// first: a skipped instance meters silence for that cycle rather than its previous block again.
struct HubKey {
    int family;                                                // lv2_shim.cu: its Kind; lv2_ebur128.cu, lv2_stats.cu: HUB_*
    int ppm_kind; uint32_t chn, tpk_flags; double rate;        // chn: staged rows per slot; HUB_DR14: tpk_flags = DR mode
    bool operator== (const HubKey& o) const
    {
        return family == o.family && ppm_kind == o.ppm_kind && chn == o.chn && tpk_flags == o.tpk_flags && rate == o.rate;
    }
};
constexpr int HUB_EBUR128 = -1, HUB_BITMETER = -2, HUB_SIGDIST = -3, HUB_DR14 = -4;

class SlotHub {
public:
    // mu guards the hub and its bank: take it for any bank call made outside submit / close_if_broken
    std::mutex mu;
    const HubKey key; const uint32_t slots;

    virtual ~SlotHub () { stage.release (); }

    // Joins `who` to a hub with this key, creating one with create (key, slots) when none has a free slot.  NULL when batched
    // mode is off or a hub cannot be made; the caller then uses a private bank.
    static SlotHub* join (const HubKey& key, void* who, int* slot, SlotHub* (*create) (const HubKey&, uint32_t))
    {
        const char* v = getenv ("B200M_LV2_BATCH");
        const int want = v ? atoi (v) : 0;
        if (want < 2) return nullptr;
        std::lock_guard<std::mutex> lk (registry_mu ());
        SlotHub* hub = nullptr;
        for (SlotHub* h : registry ()) if (h->key == key && h->members < h->slots) hub = h;
        if (!hub) {
            hub = create (key, (uint32_t)want);
            if (!hub) return nullptr;
            const uint32_t rows = hub->slots * key.chn;
            hub->stage.reserve (rows);
            if (!hub->stage.cap) { delete hub; return nullptr; }
            memset (hub->stage.data, 0, (size_t)rows * B200M_MAX_BLOCK * sizeof (float));
            registry ().push_back (hub);
        }
        std::lock_guard<std::mutex> lh (hub->mu);
        for (uint32_t i = 0; i < hub->slots; ++i)
            if (!hub->member[i]) { hub->member[i] = who; *slot = (int)i; ++hub->members; return hub; }
        return nullptr;
    }

    // The slot's rows idle on silence and its bank state is vacated; the last member out destroys the hub.
    void leave (int slot)
    {
        std::lock_guard<std::mutex> lk (registry_mu ());
        bool empty;
        {
            std::lock_guard<std::mutex> lh (mu);
            fetch ();
            if (submitted[slot]) { submitted[slot] = 0; --n_submitted; }
            member[slot] = nullptr; --members;
            vacate ((uint32_t)slot);
            zero_rows ((uint32_t)slot);
            empty = members == 0;
        }
        if (empty) {
            auto& r = registry ();
            for (size_t i = 0; i < r.size (); ++i) if (r[i] == this) { r.erase (r.begin () + i); break; }
            delete this;
        }
    }

    // With mu held.  Collects the cycle in flight; if this submission would break the contract (the slot already submitted,
    // or n differs from the open cycle's), launches and collects the open cycle as it is.
    void close_if_broken (int slot, uint32_t n)
    {
        fetch ();
        if (submitted[slot] || (cycle_n && cycle_n != n)) { launch (); fetch (); }
    }

    // With mu held, 1 <= n <= B200M_MAX_BLOCK, in[0 .. key.chn).  Stages the slot's input; the last member to submit launches
    // the cycle.  The results of the previous cycle stay readable until the next submit / close_if_broken collects this one.
    void submit (int slot, const float* const* in, uint32_t n)
    {
        close_if_broken (slot, n);
        for (uint32_t c = 0; c < key.chn; ++c) memcpy (row ((uint32_t)slot, c), in[c], n * sizeof (float));
        submitted[slot] = 1; ++n_submitted; cycle_n = n;
        if (n_submitted == members) launch ();
    }

protected:
    std::vector<void*> member;                                 // the plugin instance in each slot, or NULL
    PinnedStage stage;                                         // [slots * key.chn][B200M_MAX_BLOCK]

    SlotHub (const HubKey& k, uint32_t n_slots) : key (k), slots (n_slots), member (n_slots, nullptr), submitted (n_slots, 0) {}

    // the bank-specific hooks, all called with mu held
    virtual int launch_bank (uint32_t n) = 0;                  // process the staged cycle of n frames asynchronously; 0 = in flight
    virtual void collect () = 0;                               // wait for the cycle in flight and copy out its results
    virtual void vacate (uint32_t slot) = 0;                   // the slot's member left

private:
    std::vector<uint8_t> submitted;
    uint32_t members = 0, n_submitted = 0, cycle_n = 0;
    bool inflight = false;

    static std::mutex& registry_mu () { static std::mutex m; return m; }
    static std::vector<SlotHub*>& registry () { static std::vector<SlotHub*> r; return r; }

    float* row (uint32_t slot, uint32_t c) { return stage.data + ((size_t)slot * key.chn + c) * B200M_MAX_BLOCK; }
    void zero_rows (uint32_t slot) { memset (row (slot, 0), 0, (size_t)key.chn * B200M_MAX_BLOCK * sizeof (float)); }

    void fetch ()
    {
        if (!inflight) return;
        collect ();
        inflight = false;
    }
    void launch ()
    {
        if (n_submitted < members)
            for (uint32_t i = 0; i < slots; ++i) if (member[i] && !submitted[i]) zero_rows (i);
        inflight = cycle_n && launch_bank (cycle_n) == 0;
        std::fill (submitted.begin (), submitted.end (), 0);
        n_submitted = 0; cycle_n = 0;
    }
};

// Batched phasewheel and goniometer instances (lv2_xfer.cu, lv2_gon.cu) share the COR plugin's hub of their sample rate
// (lv2_shim.cu).  cor_hub_join: a slot cleared to a fresh Stcorrdsp, or NULL when batched mode is off; leave with hub->leave (slot).
// cor_hub_cycle: returns the slot's reading of the previous cycle and submits this cycle's n frames of in[0], in[1]; a held cycle
// leaves the slot's Stcorrdsp untouched, as a private instance that does not call process () in it.
SlotHub* cor_hub_join (double rate, void* who, int* slot);
float cor_hub_cycle (SlotHub* hub, int slot, const float* const* in, uint32_t n, bool hold);

}  // namespace b200m
