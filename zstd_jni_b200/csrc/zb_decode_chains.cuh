// zb_decode_chains.cuh -- device side of stages B + C of the staged decoder (zb_decode_fast.cuh): k_dec_chains.
//
// One persistent CTA per SM, six warps:
//   warps 0 .. 1   Huffman chains: 8 frames x 4 streams per warp (HufChain)
//   warps 2 .. 3   sequence chains, WALK half: CH_FSE_LANES lanes per warp, one frame per lane (SeqChain::walk) -- each alone
//                  on its scheduler, because a chain is as fast as its warp issues
//   warps 4 .. 5   sequence chains, VALUE half (SeqValue::take): lane l of warp 4 + w finishes what lane l of warp 2 + w
//                  walks; they share the schedulers of the Huffman warps, which mostly wait
// A walk lane hands its value lane 16-byte raw records through a 16-deep ring in shared memory: one 128-bit store / load each,
// a generation bit inside the record is the only flag (no fences on the chain), the value lane reports its progress every
// fourth record and the walk lane looks at that report before it could lap the ring.  Frame changes go through a small mailbox.
// Lanes are persistent: a lane (a group of 4 lanes for Huffman) that finishes its frame draws the next one from a
// longest-first work list while the other lanes keep stepping, so the kernel lasts (total steps / lanes) or as long
// as its longest chain, whichever is more -- not (waves x longest chain).
//
// Shared memory (~221 KB, the whole SM):
//   * per lane / frame slot the decode tables (3 FSE tables = 5 KB, one Huffman table = 4 KB), filled by bulk
//     asynchronous copies (cp.async.bulk global -> shared, completion on an mbarrier the owning lanes wait on);
//   * per lane a ring of CH_RING_GROUPS 16-byte cells of its bitstream: cp.async copies keep CH_RING_DEPTH cells
//     in flight below the reader, so the sequential, read-once compressed bytes come out of HBM hundreds of
//     cycles before the chain needs them and no chain ever waits for DRAM;
//   * one copy of the code tables (base values of the length codes).
#pragma once
#include "zb_decode_fast.cuh"

#if defined(__CUDACC__)
namespace zb {

constexpr int CH_FSE_WARPS = 2, CH_FSE_LANES = 14, CH_HUF_WARPS = 2;
constexpr int CH_WARPS = CH_HUF_WARPS + 2 * CH_FSE_WARPS;      // Huffman | walk | value
constexpr u32 CH_LINK_DEPTH = 16;                               // raw records between a walk lane and its value lane
constexpr u32 CH_LINK_BYTES = CH_LINK_DEPTH * 16 + 32;          // ring + mailbox
constexpr int CH_RING_GROUPS = 8;        // 16-byte cells per lane ring
constexpr int CH_RING_DEPTH = 4;         // cells requested below the one being read
constexpr u32 CH_FSE_SLOT = FAST_FSE_ENTRIES * 4, CH_HUF_SLOT = FAST_HUF_ENTRIES * 2;
constexpr u32 CH_OFF_HUF = CH_FSE_WARPS * CH_FSE_LANES * CH_FSE_SLOT;
constexpr u32 CH_OFF_RING = CH_OFF_HUF + CH_HUF_WARPS * 8 * CH_HUF_SLOT;
constexpr u32 CH_OFF_LINK = CH_OFF_RING + (CH_HUF_WARPS * 32 + CH_FSE_WARPS * CH_FSE_LANES) * (16 + CH_RING_GROUPS * 16);
constexpr u32 CH_OFF_CT = CH_OFF_LINK + CH_FSE_WARPS * CH_FSE_LANES * CH_LINK_BYTES;
constexpr u32 CH_OFF_BAR = CH_OFF_CT + ((sizeof(CodeTables) + 15) / 16) * 16;
constexpr u32 CH_SMEM = CH_OFF_BAR + (CH_FSE_WARPS * CH_FSE_LANES + CH_HUF_WARPS * 8) * 8;

__device__ __forceinline__ u32 smem_u32(const void* p) { return (u32)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(u32 bar, u32 count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(bar), "r"(count) : "memory"); }
__device__ __forceinline__ void mbar_expect_tx(u32 bar, u32 bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"(bytes) : "memory"); }
__device__ __forceinline__ void bulk_g2s(u32 dst, const void* src, u32 bytes, u32 bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" :: "r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(u32 bar, u32 parity) {
    u32 ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void cp_async16(u32 dst, const void* src) { asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(dst), "l"(src) : "memory"); }
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" :: "n"(N) : "memory"); }
// wait for a table copy; gives up after ~2^22 polls (a copy that never lands must not hang the device: the caller
// reports corruption for the frame instead)
__device__ __forceinline__ bool mbar_wait(u32 bar, u32 parity) {
    for (u32 spin = 0; spin < (1u << 22); spin++) if (mbar_try_wait(bar, parity)) return true;
    return false;
}

// word source of a chain on the GPU: the lane's ring.  32 words (8 groups of 16 bytes) plus a mirror cell below them that
// repeats the top group, so that the four words k, k-1, k-2, k-3 of a window are always at one address and three immediate
// offsets below it -- no wrap-around arithmetic on the chain.
constexpr u32 CH_RING_LANE_BYTES = 16 + CH_RING_GROUPS * 16;       // mirror cell + ring
constexpr u32 CH_RING_WARP_BYTES = 32 * CH_RING_LANE_BYTES;
struct RingWords {
    StreamGeom g;
    u32 ring0;           // shared-memory address of the lane's ring word 0 (the mirror cell sits 16 bytes below)
    int gIssued;         // lowest 16-byte group requested so far
    __device__ __forceinline__ u32 lds(u32 addr) const { u32 v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory"); return v; }
    __device__ __forceinline__ u32 raw(int k) const { return lds(ring0 + (((u32)k & (CH_RING_GROUPS * 4 - 1)) << 2)); }
    __device__ __forceinline__ u32 word(int k) const { return k < g.kFirst ? 0u : g.fix(k, raw(k)); }
    __device__ __forceinline__ void fetch4(int k, u32& a, u32& b, u32& c, u32& d) const {
        if (k >= 8) {                                    // kFirst <= 3: no masks up here
            u32 const at = ring0 + (((u32)k & (CH_RING_GROUPS * 4 - 1)) << 2);
            asm volatile("ld.shared.u32 %0, [%4];\n\tld.shared.u32 %1, [%4+-4];\n\tld.shared.u32 %2, [%4+-8];\n\tld.shared.u32 %3, [%4+-12];"
                         : "=r"(a), "=r"(b), "=r"(c), "=r"(d) : "r"(at) : "memory");
        } else { a = word(k); b = word(k - 1); c = word(k - 2); d = word(k - 3); }
    }
    __device__ __forceinline__ void fetch4_fast(int k, u32& a, u32& b, u32& c, u32& d) const {
        u32 const at = ring0 + (((u32)k & (CH_RING_GROUPS * 4 - 1)) << 2);
        asm volatile("ld.shared.u32 %0, [%4];\n\tld.shared.u32 %1, [%4+-4];\n\tld.shared.u32 %2, [%4+-8];\n\tld.shared.u32 %3, [%4+-12];"
                     : "=r"(a), "=r"(b), "=r"(c), "=r"(d) : "r"(at) : "memory");
    }
    // advance() without a branch: the copies are predicated, a (possibly empty) group is committed every time -- empty groups only
    // make the real requests look older to wait_group, which keeps its guarantee
    __device__ __forceinline__ void advance_fast(int k) {
        bool const need = gIssued > (k >> 2) - CH_RING_DEPTH;
        gIssued -= need ? 1 : 0;
        u32 const m = (u32)gIssued & (CH_RING_GROUPS - 1);
        u32 const p1 = (need && gIssued >= 0) ? 1u : 0u, p2 = (p1 && m == CH_RING_GROUPS - 1) ? 1u : 0u;
        asm volatile("{\n\t.reg .pred p, q;\n\tsetp.ne.u32 p, %3, 0;\n\tsetp.ne.u32 q, %4, 0;\n\t"
                     "@p cp.async.cg.shared.global [%0], [%2], 16;\n\t@q cp.async.cg.shared.global [%1], [%2], 16;\n\t"
                     "cp.async.commit_group;\n\t}"
                     :: "r"(ring0 + m * 16), "r"(ring0 - 16), "l"(g.W + 4 * gIssued), "r"(p1), "r"(p2) : "memory");
        cp_async_wait<CH_RING_DEPTH - 1>();
    }
    __device__ __forceinline__ void request_next() {    // one more group below the lowest requested one
        gIssued--;
        if (gIssued >= 0) {
            u32 const m = (u32)gIssued & (CH_RING_GROUPS - 1);
            cp_async16(ring0 + m * 16, g.W + 4 * gIssued);
            if (m == CH_RING_GROUPS - 1) cp_async16(ring0 - 16, g.W + 4 * gIssued);      // the top group also fills the mirror cell
        }
        cp_async_commit();
    }
    // the reader now stands at word k (at most one group below where it stood): keep CH_RING_DEPTH groups requested below
    // it, then make sure the group of k and the one below have landed (all but the CH_RING_DEPTH - 1 youngest requests)
    __device__ __forceinline__ void advance(int k) {
        if (gIssued > (k >> 2) - CH_RING_DEPTH) request_next();
        cp_async_wait<CH_RING_DEPTH - 1>();
    }
    __device__ __forceinline__ void start(const u8* ip, u32 bits) {
        g.set(ip);
        int const k = ((int)(g.floorBit + bits) - 1) >> 5;
        gIssued = (k >> 2) + 1;
        while (gIssued > (k >> 2) - CH_RING_DEPTH) request_next();
        cp_async_wait<CH_RING_DEPTH - 1>();
    }
};

struct ChainsArgs {
    const u8* srcBase; const u64* srcOff; u32 n; DecDesc* descs;
    const u32* fseBase; const u16* hufBase; u64* seqBase; u8* litBase; size_t litStride;
    u32* counterSeq; u32* counterHuf; const u32* orderSeq; const u32* orderHuf;
    u32 roles;           // experiments: bit 0 = run the sequence chains, bit 1 = run the Huffman chains (3 = both, the product setting)
};

// shared-memory traffic between a walk lane and its value lane (volatile: another warp is on the other side)
__device__ __forceinline__ u32 lds_v(u32 addr) { u32 v; asm volatile("ld.volatile.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory"); return v; }
__device__ __forceinline__ void sts_v(u32 addr, u32 v) { asm volatile("st.volatile.shared.u32 [%0], %1;" :: "r"(addr), "r"(v) : "memory"); }
__device__ __forceinline__ void sts_v4(u32 addr, u32 a, u32 b, u32 c, u32 d) { asm volatile("st.volatile.shared.v4.u32 [%0], {%1, %2, %3, %4};" :: "r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory"); }
__device__ __forceinline__ void lds_v4(u32 addr, u32& a, u32& b, u32& c, u32& d) { asm volatile("ld.volatile.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(a), "=r"(b), "=r"(c), "=r"(d) : "r"(addr) : "memory"); }
// mailbox words behind the ring
constexpr u32 LK_CONSUMED = CH_LINK_DEPTH * 16, LK_GEN = LK_CONSUMED + 4, LK_NBSEQ = LK_GEN + 4, LK_OUTLO = LK_NBSEQ + 4, LK_OUTHI = LK_OUTLO + 4;

__device__ __forceinline__ void chains_walk_warp(const ChainsArgs& a, unsigned char* smem, int cw, int lane) {
    if (lane >= CH_FSE_LANES) return;
    constexpr u32 MASK = (1u << CH_FSE_LANES) - 1;
    int const slot = cw * CH_FSE_LANES + lane;
    u32* const tab = reinterpret_cast<u32*>(smem + (size_t)slot * CH_FSE_SLOT);
    u32 const tabAddr = smem_u32(tab);
    u32 const bar = smem_u32(smem + CH_OFF_BAR + slot * 8);
    u32 const link = smem_u32(smem + CH_OFF_LINK + slot * CH_LINK_BYTES);
    u32 parity = 0, gen = 0, seqNo = 0, consumed = 0;
    RingWords ws; ws.ring0 = smem_u32(smem + CH_OFF_RING + (CH_HUF_WARPS * 32 + slot) * CH_RING_LANE_BYTES + 16); ws.gIssued = 0;
    SeqChain D; D.k = D.nbSeq = 0; D.top = 0; D.sLL = D.sOF = D.sML = 0;
    DecDesc* d = nullptr;
    bool live = false, exhausted = false, told = false;
    auto publish = [&](SeqRaw const& r) {
        sts_v4(link + (seqNo & (CH_LINK_DEPTH - 1)) * 16, r.v0, r.v1, r.a, (r.b & 0x7FFFFFFFu) | ((seqNo << (31 - 4)) & 0x80000000u));      // bit 31: generation of the slot
        seqNo++;
    };
    u32 consumedNext = 0;
    u32 mask = MASK;                    // lanes still at work: a lane that has run out of frames leaves, so that it cannot hold the others on the slow path
    for (;;) {
        // the common iteration: every lane in the middle of a frame with room in its ring -- one vote, then a straight line.
        // The value lane's progress report is read one iteration ahead of its use (an older report is only more cautious), so
        // the vote never waits for shared memory.
        consumed = consumedNext;
        consumedNext = lds_v(link + LK_CONSUMED);
        if (!__any_sync(mask, !live || !D.plain() || seqNo - consumed >= CH_LINK_DEPTH - 3)) {
            publish(D.walk<true>(ws, tab, tab + FAST_FSE_OF, tab + FAST_FSE_ML));
            continue;
        }
        if (!live && !exhausted) {
            u32 item = atomicAdd(a.counterSeq, 1u);
            if (item >= a.n) exhausted = true;
            else {
                item = a.orderSeq[item];
                d = a.descs + item;
                u32 const nbSeq = d->nbSeq;
                if (nbSeq == 0) exhausted = true;            // k_order puts every frame without sequences after all others: none left
                else if (d->mode == 1 && !d->stA1 && !d->stA2 && !d->seqUnusable) {
                    u32 const logLL = d->logLL, logOF = d->logOF, logML = d->logML;
                    u32 const bLL = umax(16u, 4u << logLL), bOF = umax(16u, 4u << logOF), bML = umax(16u, 4u << logML);
                    const u32* const gt = a.fseBase + (size_t)item * FAST_FSE_ENTRIES;
                    fence_proxy_async();                     // the slot's previous tables were read through the generic proxy
                    mbar_expect_tx(bar, bLL + bOF + bML);
                    bulk_g2s(tabAddr, gt, bLL, bar);
                    bulk_g2s(tabAddr + FAST_FSE_OF * 4, gt + FAST_FSE_OF, bOF, bar);
                    bulk_g2s(tabAddr + FAST_FSE_ML * 4, gt + FAST_FSE_ML, bML, bar);
                    ws.start(a.srcBase + a.srcOff[item] + d->blockOff + d->seqOff, d->seqBits);
                    // the value lane must be through with the previous frame before the mailbox changes
                    while (lds_v(link + LK_CONSUMED) != seqNo) {}
                    u64 const outp = reinterpret_cast<u64>(a.seqBase + (size_t)item * FAST_MAXS);
                    sts_v(link + LK_NBSEQ, nbSeq); sts_v(link + LK_OUTLO, (u32)outp); sts_v(link + LK_OUTHI, (u32)(outp >> 32));
                    __threadfence_block();
                    sts_v(link + LK_GEN, ++gen);
                    bool const landed = mbar_wait(bar, parity);
                    parity ^= 1;
                    if (!landed) {                           // tell the value lane to skip this frame: it sees fewer records than announced -> send zeros
                        d->stC = E_GENERIC;
                        SeqRaw z; z.v0 = z.v1 = z.a = z.b = 0;
                        for (u32 q = 0; q < nbSeq; q++) { while (seqNo - lds_v(link + LK_CONSUMED) >= CH_LINK_DEPTH - 2) {} publish(z); }
                    } else {
                        D.begin(ws, ws.g.floorBit, d->seqBits, logLL, logOF, logML, nbSeq);
                        live = true;
                    }
                }
            }
        }
        if (exhausted && !told) {                            // end of work: an empty frame in the mailbox sends the value lane home
            while (lds_v(link + LK_CONSUMED) != seqNo) {}
            sts_v(link + LK_NBSEQ, 0u);
            __threadfence_block();
            sts_v(link + LK_GEN, ++gen);
            told = true;
        }
        {   bool const finished = !live && exhausted;         // (told by now)
            u32 const gone = __ballot_sync(mask, finished);
            if (finished) return;
            mask &= ~gone; }
        if (live) {
            while (seqNo - lds_v(link + LK_CONSUMED) >= CH_LINK_DEPTH - 2) {}
            publish(D.walk<false>(ws, tab, tab + FAST_FSE_OF, tab + FAST_FSE_ML));
            if (!D.more()) { if (!D.clean(ws.g.floorBit)) d->stC = E_corruption_detected; live = false; }
        }
    }
}

__device__ __forceinline__ void chains_value_warp(const ChainsArgs& a, unsigned char* smem, int vw, int lane) {
    (void)a;
    if (lane >= CH_FSE_LANES) return;
    constexpr u32 MASK = (1u << CH_FSE_LANES) - 1;
    int const slot = vw * CH_FSE_LANES + lane;
    const CodeTables* const ct = reinterpret_cast<const CodeTables*>(smem + CH_OFF_CT);
    u32 const link = smem_u32(smem + CH_OFF_LINK + slot * CH_LINK_BYTES);
    SeqValue V; V.begin(nullptr);
    u32 seen = 0, nb = 0, cons = 0;
    bool done = false;
    u32 mask = MASK;                    // lanes still at work (a lane that was sent home leaves)
    for (;;) {
        // the common iteration: every lane inside a frame -- one vote, one ring slot each, no branch on who had news
        if (!__any_sync(mask, V.k == nb)) {
            SeqRaw r;
            lds_v4(link + (cons & (CH_LINK_DEPTH - 1)) * 16, r.v0, r.v1, r.a, r.b);
            bool const ok = (r.b >> 31) == ((cons >> 4) & 1);
            V.take_if(ok, r, ct);
            cons += ok ? 1u : 0u;
            if (ok && (cons & 3) == 0) sts_v(link + LK_CONSUMED, cons);
            continue;
        }
        if (!done) {
            if (V.k == nb) {                                 // between frames: report, then look for the next mailbox
                sts_v(link + LK_CONSUMED, cons);
                u32 const g = lds_v(link + LK_GEN);
                if (g != seen) {
                    __threadfence_block();
                    nb = lds_v(link + LK_NBSEQ);
                    u64 const outp = (u64)lds_v(link + LK_OUTLO) | ((u64)lds_v(link + LK_OUTHI) << 32);
                    V.begin(reinterpret_cast<u64*>(outp));
                    seen = g;
                    if (nb == 0) done = true;
                }
            } else {
                SeqRaw r;
                lds_v4(link + (cons & (CH_LINK_DEPTH - 1)) * 16, r.v0, r.v1, r.a, r.b);
                if ((r.b >> 31) == ((cons >> 4) & 1)) {      // the record of this turn of the ring has arrived
                    V.take(r, ct);
                    cons++;
                    if ((cons & 3) == 0) sts_v(link + LK_CONSUMED, cons);
                }
            }
        }
        {   u32 const gone = __ballot_sync(mask, done);
            if (done) return;
            mask &= ~gone; }
    }
}

__device__ __forceinline__ void chains_huf_warp(const ChainsArgs& a, unsigned char* smem, int hwarp, int lane) {
    int const grp = lane >> 2, k = lane & 3;
    u32 const gmask = 0xFu << (lane & ~3);
    int const slot = hwarp * 8 + grp;
    u16* const tab = reinterpret_cast<u16*>(smem + CH_OFF_HUF + (size_t)slot * CH_HUF_SLOT);
    u32 const tabAddr = smem_u32(tab);
    u32 const bar = smem_u32(smem + CH_OFF_BAR + (CH_FSE_WARPS * CH_FSE_LANES + slot) * 8);
    u32 parity = 0;
    RingWords ws; ws.ring0 = smem_u32(smem + CH_OFF_RING + (hwarp * 32 + lane) * CH_RING_LANE_BYTES + 16); ws.gIssued = 0;
    HufChain H; H.left = 0; H.op = nullptr; H.kNext = 0; H.hi = H.lo = 0; H.avail = 0; H.budget = 0;
    DecDesc* d = nullptr;
    u32 sh = 0;
    bool live = false, exhausted = false;
    u32 mask = 0xFFFFFFFFu;             // groups still at work: a group that has run out of frames leaves, so that it cannot hold the others on the slow path
    for (;;) {
        if (!__any_sync(mask, !live || !H.plain())) { H.step4_fast(ws, tab, sh); continue; }
        u32 const liveMask = __ballot_sync(mask, live);
        {   bool const finished = (liveMask & gmask) == 0 && exhausted;      // uniform inside a group
            u32 const gone = __ballot_sync(mask, finished);
            if (finished) return;
            mask &= ~gone; }
        if ((liveMask & gmask) == 0) {                       // the group's four streams are done: next frame
            u32 item = 0xFFFFFFFFu;
            if (k == 0) { item = atomicAdd(a.counterHuf, 1u); item = item < a.n ? a.orderHuf[item] : 0xFFFFFFFFu; }
            item = __shfl_sync(gmask, item, lane & ~3);
            if (item == 0xFFFFFFFFu) exhausted = true;
            else {
                d = a.descs + item;
                if (d->hufLitSize == 0) exhausted = true;    // k_order puts every frame without Huffman literals last: none left
                else if (d->mode == 1 && !d->stA1 && d->litMode == 2) {
                    u32 const log = d->hufLog;
                    __syncwarp(gmask);                         // the siblings' last reads of the slot's old table come first
                    if (k == 0) {
                        fence_proxy_async();
                        u32 const bytes = umax(16u, 2u << log);
                        mbar_expect_tx(bar, bytes);
                        bulk_g2s(tabAddr, a.hufBase + (size_t)item * FAST_HUF_ENTRIES, bytes, bar);
                    }
                    u32 const bits = k < (int)d->nStreams ? d->sBits[k] : HUF_UNUSABLE;
                    const u8* const blk = a.srcBase + a.srcOff[item] + d->blockOff;
                    if (bits != HUF_UNUSABLE) ws.start(blk + d->sOff[k], bits);
                    bool const landed = __all_sync(gmask, mbar_wait(bar, parity));      // (one verdict per group)
                    parity ^= 1;
                    if (!landed) { d->stB = E_GENERIC; exhausted = true; }
                    else if (bits != HUF_UNUSABLE) {
                        H.begin(ws, ws.g.floorBit, bits, a.litBase + (size_t)item * a.litStride + d->oOff[k], d->oCnt[k]);
                        sh = 32 - log;
                        live = H.left != 0;
                        if (!live && !H.clean()) d->stB = E_corruption_detected;
                    }
                }
            }
        }
        if (live) {
            if (H.left >= 4 && H.aligned4()) H.step4(ws, tab, sh); else H.step1(ws, tab, sh);
            if (H.left == 0) { if (!H.clean()) d->stB = E_corruption_detected; live = false; }
        }
    }
}

__global__ void __launch_bounds__(CH_WARPS * 32, 1) k_dec_chains(ChainsArgs a) {
    extern __shared__ __align__(128) unsigned char smem[];
    int const warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    {   const u32* const srcw = reinterpret_cast<const u32*>(&c_tables); u32* const dstw = reinterpret_cast<u32*>(smem + CH_OFF_CT);
        for (u32 j = threadIdx.x; j < sizeof(CodeTables) / 4; j += blockDim.x) dstw[j] = srcw[j]; }
    if (threadIdx.x == 0) {
        for (int j = 0; j < CH_FSE_WARPS * CH_FSE_LANES + CH_HUF_WARPS * 8; j++) mbar_init(smem_u32(smem + CH_OFF_BAR + j * 8), 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    // links: every ring slot starts in the "other" generation, mailboxes empty
    for (u32 j = threadIdx.x; j < CH_FSE_WARPS * CH_FSE_LANES * (CH_LINK_BYTES / 4); j += blockDim.x) {
        u32 const wIn = j % (CH_LINK_BYTES / 4);
        reinterpret_cast<u32*>(smem + CH_OFF_LINK)[j] = wIn < CH_LINK_DEPTH * 4 ? 0xFFFFFFFFu : 0u;
    }
    __syncthreads();
    if (warp < CH_HUF_WARPS) { if (a.roles & 2) chains_huf_warp(a, smem, warp, lane); }
    else if (warp < CH_HUF_WARPS + CH_FSE_WARPS) { if (a.roles & 1) chains_walk_warp(a, smem, warp - CH_HUF_WARPS, lane); }
    else if (a.roles & 1) chains_value_warp(a, smem, warp - CH_HUF_WARPS - CH_FSE_WARPS, lane);
}

}  // namespace zb
#endif
