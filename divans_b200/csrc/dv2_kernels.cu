// dv2_kernels.cu -- stream decoder of the v2 engine (dv2_core.cuh): persistent warps, every warp runs 32 / LPG streams in
// lock step (LPG = 16: two, LPG = 8: four), work pulled from a global counter.  Same framing pre-pass (dv_kernels.cu) and
// the same command state machine (dv_engine_kernel.cuh, transition<false, true>) as the blend decoder and the encoder.
#include "dv2_core.cuh"

namespace dv {

constexpr int DEC2_BLOCK_THREADS = 32;          // one warp per block: blocks spread evenly over the SMs
constexpr int DEC2_MIN_BLOCKS = 16;             // 4 one-warp blocks per scheduler partition (16 K registers each): <= 128 registers, 32 resident
                                                // 16-lane streams per SM (4224 on an H100's 132 SMs).  (144 registers = 3 per partition = 12 per
                                                // SM: 3168 resident 16-lane streams, a second wave for 4096)

template <int LPG>
__global__ void __launch_bounds__(DEC2_BLOCK_THREADS, DEC2_MIN_BLOCKS) decode_kernel_v2(DecodeParams p) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int lane = threadIdx.x & 31;
    const int warp_in_block = threadIdx.x >> 5;
    constexpr int GPW = 32 / LPG;
    const int group_in_block = warp_in_block * GPW + lane / LPG;
    // behind the groups' cold state: 16 lanes per stream, each group's T2S (dv2_core.cuh)
    constexpr uint32_t T2S_OFF = (DEC2_BLOCK_THREADS / LPG) * SMEM_BYTES_PER_GROUP_V2;
    const uint32_t t2s = LPG == 16 ? (uint32_t)__cvta_generic_to_shared(smem + T2S_OFF) + (uint32_t)group_in_block * T2S_BYTES : 0u;
    const uint32_t slot = blockIdx.x * (DEC2_BLOCK_THREADS / LPG) + group_in_block;
    G2 g;
    g.l16 = lane & (LPG - 1);
    g.shift = lane & ~(LPG - 1);
    g.gmask = (LPG == 16 ? 0xffffu : 0xffu) << g.shift;
    g.store0 = g.l16 == 0;
    g.nl = LPG;
    g.grp = group_in_block;
    g.blend = false;

    St s;
    {   // (kept opaque: the compiler would rather rebuild this pointer from blockIdx and the parameter block at the head of
        // every iteration -- seven instructions -- than hold it)
        unsigned long long sp = reinterpret_cast<unsigned long long>(p.arena + (uint64_t)slot * SLOT_STRIDE);
        asm volatile("" : "+l"(sp));
        s.slot = reinterpret_cast<uint8_t *>(sp);
    }
    s.c = reinterpret_cast<Cold *>(smem + group_in_block * SMEM_BYTES_PER_GROUP_V2);
    s.tables = p.tables;
    s.state = S_IDLE;
    s.c->desired_context_mixing = 0; s.c->desired_prior_depth = 0; s.c->desired_force_stride = 9; s.c->desired_do_context_map = true;
    s.c->have_desired_adapt = false; s.c->desired_adapt0 = s.c->desired_adapt1 = s.c->desired_adapt2 = s.c->desired_adapt3 = 0;
    s.c->in.cmds = nullptr; s.c->in.n_cmds = 0; s.c->in.pos = 0; s.c->in.n_pms = 0; s.c->in.pms = nullptr; s.c->in.lits = nullptr;
    s.c->model_rev = p.model_rev;
    s.c->sidx = 0; s.out = nullptr; s.out_pos = 0; s.c->out_cap = 0; s.c->ring_len = 1024;
    s.c->gen_ctr = *reinterpret_cast<const uint32_t *>(s.slot + OFF_HDR);   // generations survive from launch to launch
    s.gen = 0;
    st_reset(s);
    coder_init_dec(s.cur, nullptr, 0); s.cur.need_a = 0; coder_init_dec(s.c->oth, nullptr, 0);
    Next nx; nx.cdf = A_misc(s, MI_DUMMY); nx.cdf2 = nullptr; nx.speed = SPK_NONE; nx.sym = 0; nx.mix_hi = false; nx.tagged = false;
    store_default_cdfs(g, reinterpret_cast<int16_t *>(s.slot + OFF_MISC), (uint32_t)MISC_CDFS);   // incl. the dummy CDF
    constexpr int S_DONE = -1;   // idle and the work queue is empty (v2 kernel only; one register less than a separate flag)

    for (;;) {
        __syncwarp();
        // ---- fetch work for idle groups (converged; the broadcast shuffle is executed by every lane) ----
        const bool want = s.state == S_IDLE;
        if (__any_sync(FULL, want)) {
            uint32_t v = 0;
            if (want && g.store0) v = atomicAdd(p.work_counter, 1u);
            v = __shfl_sync(FULL, v, 0, LPG);
            if (want) {
                if (v >= p.n_streams) s.state = S_DONE;
                else if (p.status[v] != ST_OK) { if (g.store0) p.out_len[v] = 0; }   // framing / CRC failure: stay idle, fetch again
                else {
                    const uint8_t *in = p.in + p.in_off[v];
                    const uint32_t pay0 = p.frame[4 * v + 1], pay1 = p.frame[4 * v + 2];
                    const uint8_t *pl = p.payload + 16ull * p.frame[4 * v + 3];
                    s.c->sidx = v;
                    s.out = p.out + p.out_off[v];
                    uint64_t cap = p.out_cap[v];
                    s.c->out_cap = cap > 0xffffffffull ? 0xffffffffu : (uint32_t)cap; s.out_pos = 0;
                    s.c->ring_len = 1u << in[5];
                    reset_slot_v2(g, s.slot);
                    st_reset(s);
                    // a new generation: every literal prior of the slot reads as the default CDF until this stream writes it.  The
                    // tables are wiped when the 16-bit generation wraps, or when an earlier user of the slot (a stream with
                    // wrapping speeds, in any engine) may have left elements that use their sign bits
                    uint32_t *hdr = reinterpret_cast<uint32_t *>(s.slot + OFF_HDR);
                    uint32_t ctr = s.c->gen_ctr + 1;
                    if ((ctr & 0xffffu) == 0 || hdr[1] != 0) {
                        v2_clear_literal_tables(g, s.slot);
                        if (g.store0) hdr[1] = 0;
                        if ((ctr & 0xffffu) == 0) ctr++;
                    }
                    s.c->gen_ctr = ctr; s.gen = ctr & 0xffffu;
                    coder_init_dec(s.cur, reinterpret_cast<const uint32_t *>(pl), pay0 >> 2);   // command stream (CMD_CODER, codec/interface.rs:49)
                    coder_init_dec(s.c->oth, reinterpret_cast<const uint32_t *>(pl + (((uint64_t)pay0 + 15) & ~15ull)), pay1 >> 2);   // literal stream (LIT_CODER, :50)
                    enter_cmd_type<false>(s, nx);
                }
            }
            if (__all_sync(FULL, s.state == S_DONE)) break;
            __syncwarp();
        }
        // ---- whole literal bytes while every group is at a byte boundary of a literal (or out of work) ----
        const bool lit = s.state == S_LIT_HI;
        if (__any_sync(FULL, lit) && __all_sync(FULL, lit || s.state == S_DONE) && literal_fast_v2<LPG>(s, nx, g, lit, t2s)) {   // (the cheaper, usually false test first)
            if (lit) {
                if (s.cur.underflow) s.status = ST_NEED_INPUT;
                if (s.lit_left == 0 && s.status == ST_OK) { swap_coders(s, g); enter_cmd_type<false>(s, nx); }
                if (s.status != ST_OK) {
                    if (g.store0) { p.out_len[s.c->sidx] = s.out_pos; p.status[s.c->sidx] = s.status; }
                    s.state = S_IDLE; s.status = ST_OK;
                    nx.cdf = A_misc(s, MI_DUMMY); nx.cdf2 = nullptr; nx.speed = SPK_NONE; nx.tagged = false;
                    coder_init_dec(s.cur, nullptr, 0); s.cur.need_a = 0;
                }
            }
            continue;
        }
        // ---- one nibble per group ----
        const bool busy = s.state > S_IDLE;
        const int sym = nibble_core_v2<LPG>(s, nx, g);
        // ---- per-group scalar state machines (divergent) ----
        if (busy) {
            if (s.cur.underflow) s.status = ST_NEED_INPUT;
            else transition<false, true>(s, nx, g, sym);
            if (s.status != ST_OK || s.state == S_IDLE) {
                if (s.status == ST_OK && s.c->oth.underflow) s.status = ST_NEED_INPUT;
                if (g.store0) { p.out_len[s.c->sidx] = s.out_pos; p.status[s.c->sidx] = s.status; }
                s.state = S_IDLE; s.status = ST_OK;
                nx.cdf = A_misc(s, MI_DUMMY); nx.cdf2 = nullptr; nx.speed = SPK_NONE; nx.tagged = false;
                coder_init_dec(s.cur, nullptr, 0); s.cur.need_a = 0;
            }
        }
    }
    if (g.store0) *reinterpret_cast<uint32_t *>(s.slot + OFF_HDR) = s.c->gen_ctr;
}

// per block: the groups' cold state, 16 lanes per stream their T2S
template <int LPG> static size_t smem_v2() {
    return (size_t)(DEC2_BLOCK_THREADS / LPG) * (SMEM_BYTES_PER_GROUP_V2 + (LPG == 16 ? T2S_BYTES : 0));
}
template <int LPG> static void launch_v2(const DecodeParams &p, uint32_t n_blocks, cudaStream_t st) {
    decode_kernel_v2<LPG><<<n_blocks, DEC2_BLOCK_THREADS, smem_v2<LPG>(), st>>>(p);
}
template <int LPG> static int max_blocks_v2() { return stream_kernel_blocks_per_sm(decode_kernel_v2<LPG>, DEC2_BLOCK_THREADS, smem_v2<LPG>()); }
void launch_decode_v2(int lanes_per_stream, const DecodeParams &p, uint32_t n_blocks, cudaStream_t st) {
    if (lanes_per_stream == 8) launch_v2<8>(p, n_blocks, st); else launch_v2<16>(p, n_blocks, st);
}
int decode_max_blocks_per_sm_v2(int lanes_per_stream) { return lanes_per_stream == 8 ? max_blocks_v2<8>() : max_blocks_v2<16>(); }
int decode_groups_per_block_v2(int lanes_per_stream) { return DEC2_BLOCK_THREADS / lanes_per_stream; }

}  // namespace dv
