// sweep_lstm.cu -- the LSTM recurrences of a temporal layer (cell = 1, include/ctcb200.h) as ONE persistent kernel.
//
// Per direction, with z = pre + U h_prev in gate order i, f, g, o (torch.nn.LSTM's):
//   forward : i, f, o = sigmoid(z_i, z_f, z_o), g = tanh(z_g);  c = f c_prev + i g;  h = o tanh(c)
//   BPTT    : dh = delta + U^T dz_next;  dc = dh o (1 - tanh^2 c) + dc_next f_next;
//             dz = [dc g i(1-i), dc c_prev f(1-f), dc i (1-g^2), dh tanh(c) o(1-o)]
// h, c, dz and dc are 0 at every frame t >= T_u, so the backward-in-time direction starts at T_u - 1.
//
// Design: the generic sweep's (sweep.cu) with the rows regrouped.  A CTA of 8 warps owns 8 hidden units; warp w keeps
// the FOUR gate rows of unit j0 + w (forward: rows U[r H + j][:], BPTT: the columns U[r H + :][j] of the four gate
// blocks), so after the transposing butterfly lane (r, b) holds gate r -- or, in BPTT, the part of dh that gate block r
// contributes -- of utterance b, and the cell update is four shuffles inside the warp: no second exchange per step.
// The state of the previous step (h, or the dz of all 4H rows in BPTT) is exchanged through L2, as the generic sweep
// does.  U lives in registers where the CTAs that hold it are co-resident (H = 64..1024 in steps of powers of two,
// while ndir * H / 8 CTAs fit one per SM), else it is re-read through L1/L2.
//
// From coop_sweep.cuh, which the generic sweep shares: the block and tile sizes, the state-tile load, the transposing
// butterfly, the partition's tiles, the bounded step barrier (a timeout sets the error flag to 4 and the sweep runs on),
// and on the host the partition planner, the KI dispatch and the cooperative launch.
//
// The forward mode writes the activated gates over the pre-activations in place, c of every frame, and h into the
// layer's For / Back; the BPTT mode reads those back and carries dc from step to step in a [B][H] scratch per direction.
//
// Peephole mode (PEEP, include/ctcb200.h: peephole = 1): z_i and z_f also get p_i c_prev and p_f c_prev, and z_o gets
// p_o c, so the output gate is activated behind the cell update.  Every term is element-wise in the warp that owns the
// unit.  BPTT: dc = dh o (1 - tanh^2 c) + p_o dz_o + carry, and the scratch carries f dc + p_i dz_i + p_f dz_f of the
// step just finished instead of dc.  The peephole weight gradients are a separate reduction over dz and c
// (lstm_peephole_grad below).
//
// Zoneout mode (ZO, include/ctcb200.h: zoneout = 1), composed with either: after the cell update c_t and h_t each keep
// the previous step's value where their mask says so (a select, so a kept value has the bytes of c_{t-1} / h_{t-1}),
// or, in expectation mode, become the z-weighted blend.  The masks are one Philox block per (t, b, j), drawn by every
// lane of the warp for its utterance ob, and are drawn again in BPTT rather than stored: the draw is a few dozen
// integer instructions per step and lane, a stored mask would be a pass, a buffer and a load per step.  BPTT carries
// lambda_h dh in a second [ndir][B][H] scratch and, as PEEP does, the whole dc_{t+1} term of dc_t in the first.
#include "coop_sweep.cuh"
#include <cmath>
#include <curand_philox4x32_x.h>

namespace ctcb {

constexpr int LS_UNITS = 8;    // hidden units per CTA (one per warp, four gate rows each)

struct LstmArgs {
    int mode;                  // 0: forward recurrences, 1: BPTT
    int T, B, H;
    const int32_t *Tlen;       // [B]
    float *gates;              // [T][B][G], G = ndir 4H: mode 0 pre-activations in, activated gates out; mode 1 in
    const float *U[2];         // 4H x H per direction, row-major (gate row x unit)
    float *h[2];               // mode 0: [T][B][H] out
    float *c[2];               // [T][B][H]: mode 0 out, mode 1 in
    const float *dh;           // mode 1: [T][B][H], the gradient w.r.t. the layer's output
    float *dz;                 // mode 1: [T][B][G] out
    float *dc;                 // mode 1: [ndir][B][H] carry
    int parts;                 // utterance partitions (gridDim.y)
    int ndir;
    unsigned int *err;         // word 0 of the scratch: the error flag, cleared by the caller
    unsigned int *counters;    // [ndir * parts], zeroed before the launch
};
// peephole mode: the three peephole vectors of each direction, [3][H] (rows i, f, o)
struct LstmPeepArgs : LstmArgs {
    const float *P[2];
};
// zoneout mode: the probabilities, the draw and the dh carry (P is null without peepholes)
struct LstmZoArgs : LstmPeepArgs {
    float *dhc;                // mode 1: [ndir][B][H] carry, lambda_h dh of the step just finished
    int train;                 // 1: masks drawn from Philox; 0: the expectation, lambda = z
    float zc, zh;              // expectation mode
    uint32_t thr_c, thr_h;     // training mode: keep iff r < thr
    uint2 key;
    const int64_t *step;       // training mode: the device step counter
    int64_t first, stride;     // utterance b of the call is minibatch utterance first + stride b
    int layer;                 // the hidden-layer index of the temporal layer, 1..255
};
template <bool PEEP, bool ZO> struct LstmArgsOf { using type = LstmArgs; };
template <> struct LstmArgsOf<true, false> { using type = LstmPeepArgs; };
template <bool PEEP> struct LstmArgsOf<PEEP, true> { using type = LstmZoArgs; };

__device__ __forceinline__ float lstm_sigmoid(float z) { return 1.f / (1.f + expf(-z)); }

// zoneout of one state value: training mode selects prev where the mask keeps it, expectation mode blends with lambda = z
__device__ __forceinline__ float zone(const LstmZoArgs &a, bool keep, float z, float prev, float cur) {
    return a.train ? (keep ? prev : cur) : fmaf(z, prev, (1.f - z) * cur);
}

// KI > 0: H == 32 KI and U lives in registers (one CTA per SM).  KI == 0: any H, U re-read (two CTAs per SM).
template <int KI, bool PEEP, bool ZO>
__global__ void __launch_bounds__(COOP_THREADS, KI > 0 ? 1 : 2) lstm_sweep_kernel(typename LstmArgsOf<PEEP, ZO>::type a) {
    extern __shared__ __align__(16) float hs[];   // [COOP_NB][Hp]
    const int H = a.H, B = a.B, T = a.T;
    const int64_t G = (int64_t)a.ndir * 4 * H;
    const int Hp = coop_hp(H);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int dir = blockIdx.z;
    const int j = blockIdx.x * LS_UNITS + warp;     // this warp's hidden unit
    const bool bptt = (a.mode == 1);
    const bool ascending = (dir == 0) != bptt;      // time runs forward for (forward, dir 0) and (BPTT, dir 1)
    const float *U = a.U[dir];
    const int64_t gbase = (int64_t)dir * 4 * H;     // this direction's gate block inside a row of G
    float wreg[4][KI > 0 ? KI : 1];
    if (KI > 0) {
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int i = 0; i < KI; ++i) {
                const int k = lane + 32 * i;
                wreg[r][i] = (j < H) ? (bptt ? U[(int64_t)(r * H + k) * H + j] : U[(int64_t)(r * H + j) * H + k]) : 0.f;
            }
    }
    int tile_beg, tile_end;
    coop_tile_range(B, a.parts, tile_beg, tile_end);
    unsigned int *ctr = a.counters + (dir * a.parts + blockIdx.y);
    const unsigned int nslices = gridDim.x;
    bool dead = false;

    // lane -> (gate r, utterance b) of the value it owns after the butterfly
    const int orow = lane >> 3, ob = lane & 7;
    float pi = 0.f, pf = 0.f, po = 0.f;     // peephole weights of unit j
    if constexpr (PEEP) {
        if (j < H) {
            const float *P = a.P[dir];
            pi = __ldg(P + j);
            pf = __ldg(P + H + j);
            po = __ldg(P + 2 * H + j);
        }
    }
    uint32_t s32 = 0;
    if constexpr (ZO) {
        if (a.train) s32 = (uint32_t)__ldg(a.step);
    }

    for (int s = 0; s < T; ++s) {
        const int t = ascending ? s : T - 1 - s;
        const int tp = (dir == 0) ? t - 1 : t + 1;     // predecessor of t in the forward recurrence
        const int tn = (dir == 0) ? t + 1 : t - 1;     // its successor: the step BPTT came from
        for (int tile = tile_beg; tile < tile_end; ++tile) {
            const int b0 = tile * COOP_NB;
            const int b = b0 + ob;
            const bool valid = (j < H) && (b < B);
            const int64_t go = ((int64_t)t * B + b) * G + gbase + (int64_t)orow * H + j;    // this lane's gate
            float gv = 0.f;
            int Tb = 0;
            if (valid) {
                gv = __ldg(a.gates + go);      // mode 0: pre-activation; mode 1: activated gate
                Tb = __ldg(a.Tlen + b);
            }
            float acc[32];
#pragma unroll
            for (int i = 0; i < 32; ++i) acc[i] = 0.f;
            if (s > 0) {
                const int nb = min(COOP_NB, B - b0);
                if (!bptt) {       // U h_prev: the four gate rows of unit j
                    coop_load_state(hs, Hp, a.h[dir] + ((int64_t)tp * B + b0) * H, H, nb, H);
                    __syncthreads();
                    if (KI > 0) {
#pragma unroll
                        for (int i = 0; i < KI; ++i) {
                            float hv[COOP_NB];
#pragma unroll
                            for (int bb = 0; bb < COOP_NB; ++bb) hv[bb] = hs[bb * Hp + lane + 32 * i];
#pragma unroll
                            for (int r = 0; r < 4; ++r)
#pragma unroll
                                for (int bb = 0; bb < COOP_NB; ++bb) acc[r * 8 + bb] = fmaf(wreg[r][i], hv[bb], acc[r * 8 + bb]);
                        }
                    } else if (j < H) {
                        for (int k = lane; k < H; k += 32) {
                            float hv[COOP_NB], wv[4];
#pragma unroll
                            for (int bb = 0; bb < COOP_NB; ++bb) hv[bb] = hs[bb * Hp + k];
#pragma unroll
                            for (int r = 0; r < 4; ++r) wv[r] = __ldg(U + (int64_t)(r * H + j) * H + k);
#pragma unroll
                            for (int r = 0; r < 4; ++r)
#pragma unroll
                                for (int bb = 0; bb < COOP_NB; ++bb) acc[r * 8 + bb] = fmaf(wv[r], hv[bb], acc[r * 8 + bb]);
                        }
                    }
                    __syncthreads();   // hs is reused by the next tile
                } else {           // U^T dz_next, one gate block r at a time: row r of the warp sums block r
#pragma unroll
                    for (int r = 0; r < 4; ++r) {
                        coop_load_state(hs, Hp, a.dz + ((int64_t)tn * B + b0) * G + gbase + (int64_t)r * H, G, nb, H);
                        __syncthreads();
                        if (KI > 0) {
#pragma unroll
                            for (int i = 0; i < KI; ++i)
#pragma unroll
                                for (int bb = 0; bb < COOP_NB; ++bb)
                                    acc[r * 8 + bb] = fmaf(wreg[r][i], hs[bb * Hp + lane + 32 * i], acc[r * 8 + bb]);
                        } else if (j < H) {
                            for (int k = lane; k < H; k += 32) {
                                const float wv = __ldg(U + (int64_t)(r * H + k) * H + j);
#pragma unroll
                                for (int bb = 0; bb < COOP_NB; ++bb) acc[r * 8 + bb] = fmaf(wv, hs[bb * Hp + k], acc[r * 8 + bb]);
                            }
                        }
                        __syncthreads();
                    }
                }
                coop_butterfly(acc, lane);
            }
            const bool live = valid && t < Tb;
            const int64_t hc = ((int64_t)t * B + b) * H + j;      // (t, b, j) in the [T][B][H] arrays
            bool kc = false, kh = false;     // zoneout, training mode: c_t / h_t keep the previous step's value
            if constexpr (ZO) {
                if (a.train && valid) {
                    const uint32_t g = (uint32_t)(a.first + a.stride * b);
                    const uint4 r = curand_Philox4x32_10(
                        make_uint4(s32, g, (uint32_t)t, ((uint32_t)a.layer << 24) | ((uint32_t)dir << 23) | (uint32_t)j),
                        a.key);
                    kc = r.x < a.thr_c;
                    kh = r.y < a.thr_h;
                }
            }
            if (!bptt && PEEP) {
                // c_prev of utterance b from the lane that wrote it, to the four gate lanes of b
                const float cp0 = (valid && orow == 0 && live && s > 0) ? a.c[dir][((int64_t)tp * B + b) * H + j] : 0.f;
                const float cp = __shfl_sync(0xffffffffu, cp0, ob);
                float z = gv + acc[0];
                if (orow == 0) z = fmaf(pi, cp, z);
                if (orow == 1) z = fmaf(pf, cp, z);
                float act = (orow == 2) ? tanhf(z) : lstm_sigmoid(z);
                const float gi = __shfl_sync(0xffffffffu, act, ob), gf = __shfl_sync(0xffffffffu, act, 8 + ob);
                const float gg = __shfl_sync(0xffffffffu, act, 16 + ob);
                float cn = fmaf(gf, cp, gi * gg);
                if constexpr (ZO) cn = zone(a, kc, a.zc, cp, cn);
                if (orow == 3) act = lstm_sigmoid(fmaf(po, cn, z));
                const float gO = __shfl_sync(0xffffffffu, act, 24 + ob);
                if (valid) {
                    a.gates[go] = live ? act : 0.f;
                    if (orow == 0) {
                        float hn = gO * tanhf(cn);
                        if constexpr (ZO) hn = zone(a, kh, a.zh, (live && s > 0) ? a.h[dir][((int64_t)tp * B + b) * H + j] : 0.f, hn);
                        a.c[dir][hc] = live ? cn : 0.f;
                        a.h[dir][hc] = live ? hn : 0.f;
                    }
                }
            } else if (!bptt) {
                const float z = gv + acc[0];
                const float act = (orow == 2) ? tanhf(z) : lstm_sigmoid(z);
                const float gi = __shfl_sync(0xffffffffu, act, ob), gf = __shfl_sync(0xffffffffu, act, 8 + ob);
                const float gg = __shfl_sync(0xffffffffu, act, 16 + ob), gO = __shfl_sync(0xffffffffu, act, 24 + ob);
                if (valid) {
                    a.gates[go] = live ? act : 0.f;
                    if (orow == 0) {
                        const float cp = (live && s > 0) ? a.c[dir][((int64_t)tp * B + b) * H + j] : 0.f;
                        float cn = fmaf(gf, cp, gi * gg);
                        if constexpr (ZO) cn = zone(a, kc, a.zc, cp, cn);
                        float hn = gO * tanhf(cn);
                        if constexpr (ZO) hn = zone(a, kh, a.zh, (live && s > 0) ? a.h[dir][((int64_t)tp * B + b) * H + j] : 0.f, hn);
                        a.c[dir][hc] = live ? cn : 0.f;
                        a.h[dir][hc] = live ? hn : 0.f;
                    }
                }
            } else {
                const float p0 = __shfl_sync(0xffffffffu, acc[0], ob), p1 = __shfl_sync(0xffffffffu, acc[0], 8 + ob);
                const float p2 = __shfl_sync(0xffffffffu, acc[0], 16 + ob), p3 = __shfl_sync(0xffffffffu, acc[0], 24 + ob);
                const float gi = __shfl_sync(0xffffffffu, gv, ob), gf = __shfl_sync(0xffffffffu, gv, 8 + ob);
                const float gg = __shfl_sync(0xffffffffu, gv, 16 + ob), gO = __shfl_sync(0xffffffffu, gv, 24 + ob);
                if constexpr (ZO) {
                    if (valid && orow == 0) {
                        float *dcp = a.dc + ((int64_t)dir * B + b) * H + j;
                        float *dhp = a.dhc + ((int64_t)dir * B + b) * H + j;
                        // hcar: lambda_h dh, -0 where nothing is carried (x + -0 is x, bit for bit, for every x)
                        float dzi = 0.f, dzf = 0.f, dzg = 0.f, dzo = 0.f, dct = 0.f, hcar = -0.f;
                        if (live) {
                            float dh = __ldg(a.dh + hc) + ((p0 + p1) + (p2 + p3));
                            const bool has_prev = (tp >= 0 && tp < T), has_next = (s > 0);
                            if (has_next) dh += *dhp;
                            const float ct = a.c[dir][hc], tc = tanhf(ct);
                            const float cp = has_prev ? a.c[dir][((int64_t)tp * B + b) * H + j] : 0.f;
                            const float dht = a.train ? (kh ? 0.f : dh) : (1.f - a.zh) * dh;     // d h~_t
                            dzo = dht * tc * (gO * (1.f - gO));
                            const float carry = has_next ? *dcp : 0.f;
                            if constexpr (PEEP) dct = fmaf(po, dzo, dht * gO * (1.f - tc * tc)) + carry;
                            else dct = dht * gO * (1.f - tc * tc) + carry;
                            const float dcc = a.train ? (kc ? 0.f : dct) : (1.f - a.zc) * dct;     // d c~_t
                            dzi = dcc * gg * (gi * (1.f - gi));
                            dzf = dcc * cp * (gf * (1.f - gf));
                            dzg = dcc * gi * (1.f - gg * gg);
                            hcar = a.train ? (kh ? dh : -0.f) : a.zh * dh;
                        }
                        // the whole dc_t term of dc_{t-1}: (lambda_c + (1 - lambda_c) f) dc [+ p_i dz_i + p_f dz_f]
                        const float fz = a.train ? (kc ? 1.f : gf) : fmaf(1.f - a.zc, gf, a.zc);
                        if constexpr (PEEP) *dcp = (a.train && kc) ? dct : fmaf(fz, dct, fmaf(pi, dzi, pf * dzf));
                        else *dcp = (a.train && kc) ? dct : fz * dct;
                        *dhp = hcar;
                        float *dzp = a.dz + ((int64_t)t * B + b) * G + gbase + j;
                        dzp[0] = dzi;
                        dzp[H] = dzf;
                        dzp[2 * H] = dzg;
                        dzp[3 * H] = dzo;
                    }
                } else if (valid && orow == 0) {
                    float *dcp = a.dc + ((int64_t)dir * B + b) * H + j;
                    float dzi = 0.f, dzf = 0.f, dzg = 0.f, dzo = 0.f, dct = 0.f;
                    if (live) {
                        const float dh = __ldg(a.dh + hc) + ((p0 + p1) + (p2 + p3));
                        const float ct = a.c[dir][hc], tc = tanhf(ct);
                        const bool has_prev = (tp >= 0 && tp < T), has_next = (s > 0);
                        const float cp = has_prev ? a.c[dir][((int64_t)tp * B + b) * H + j] : 0.f;
                        if constexpr (PEEP) {     // the scratch holds the whole carry of the step after t
                            dzo = dh * tc * (gO * (1.f - gO));
                            const float carry = has_next ? *dcp : 0.f;
                            dct = fmaf(po, dzo, dh * gO * (1.f - tc * tc)) + carry;
                        } else {
                            const float carry = has_next ? *dcp * a.gates[((int64_t)tn * B + b) * G + gbase + H + j] : 0.f;
                            dct = dh * gO * (1.f - tc * tc) + carry;
                        }
                        dzi = dct * gg * (gi * (1.f - gi));
                        dzf = dct * cp * (gf * (1.f - gf));
                        dzg = dct * gi * (1.f - gg * gg);
                        if constexpr (!PEEP) dzo = dh * tc * (gO * (1.f - gO));
                    }
                    if constexpr (PEEP) *dcp = fmaf(gf, dct, fmaf(pi, dzi, pf * dzf));
                    else *dcp = dct;
                    float *dzp = a.dz + ((int64_t)t * B + b) * G + gbase + j;
                    dzp[0] = dzi;
                    dzp[H] = dzf;
                    dzp[2 * H] = dzg;
                    dzp[3 * H] = dzo;
                }
            }
        }
        if (s + 1 < T) coop_barrier(ctr, nslices * (unsigned int)(s + 1), a.err, 4u, dead);
    }
}

// The launch of (H, B, ndir): register-resident U where its CTAs fit one per SM, else U re-read at two CTAs per SM.
struct LstmPlan {
    int KI, parts;
    int per_sm;                // CTAs of this kernel one SM holds
    size_t smem;
};

// the plan of the kernel that runs: the peephole and zoneout modes' occupancy is their own.  CTCB_LSTM=reread takes KI = 0 at any
// H; CTCB_LSTM_PARTS forces the partition count, refused here, before any launch, where its CTAs cannot all be
// co-resident.  A width whose shared memory exceeds the opt-in maximum is refused before the attribute call.
int lstm_plan(int H, int B, int ndir, bool peep, bool zo, LstmPlan *p) {
    if (H <= 0 || B <= 0 || (ndir != 1 && ndir != 2))
        return set_error(CTCB_EINVAL, "LSTM sweep: bad sizes (H=%d, B=%d, ndir=%d)", H, B, ndir);
    const int slices = (H + LS_UNITS - 1) / LS_UNITS;
    p->smem = coop_smem(H);
    if (p->smem > max_smem_optin())
        return set_error(CTCB_EINVAL, "LSTM sweep: layerSize %d needs %zu bytes of shared memory per CTA, device allows "
                         "%zu", H, p->smem, max_smem_optin());
    const bool reg = (H == 64 || H == 128 || H == 256 || H == 512 || H == 1024) && knob(KNOB_LSTM) == 0;
    for (p->KI = reg ? H / 32 : 0;; p->KI = 0) {   // U does not fit the register files the device holds: re-read it
        const int rc = with_ki<2, 4, 8, 16, 32>(p->KI, [&](auto ki) {
            constexpr int KI = decltype(ki)::value;
            if (zo)
                return peep ? coop_occupancy(lstm_sweep_kernel<KI, true, true>, p->smem, &p->per_sm)
                            : coop_occupancy(lstm_sweep_kernel<KI, false, true>, p->smem, &p->per_sm);
            return peep ? coop_occupancy(lstm_sweep_kernel<KI, true, false>, p->smem, &p->per_sm)
                        : coop_occupancy(lstm_sweep_kernel<KI, false, false>, p->smem, &p->per_sm);
        });
        if (rc != CTCB_OK) return rc;
        if (p->KI == 0 || ndir * slices <= p->per_sm * num_sms()) break;
    }
    return coop_parts("LSTM sweep", H, p->per_sm, ndir, slices, B, knob(KNOB_LSTM_PARTS), "CTCB_LSTM_PARTS", &p->parts);
}

// ctcb_brnn_create's check that the device holds the sweep of a config
int lstm_check(int H, int B, int ndir, bool peep, bool zo) {
    if (no_device()) return CTCB_OK;
    LstmPlan p;
    return lstm_plan(H, B, ndir, peep, zo, &p);
}

size_t lstm_carry_bytes(int H, int B) { return align_up((size_t)2 * B * H * sizeof(float), 256); }

// keep iff r < floor(z 2^32), the product in float64; z in [0, 1) keeps it below 2^32
uint32_t zoneout_threshold(float z) { return (uint32_t)std::floor((double)z * 4294967296.0); }

// counters: 4096 bytes of device scratch (word 0 = error flag, cleared by the caller); dc: lstm_carry_bytes(H, B).
// Pf (and Pb with Ub) non-null: the peephole mode.  zo non-null: the zoneout mode (its dhc another
// lstm_carry_bytes(H, B) in mode 1).
int run_lstm_sweep(int mode, int T, int B, int H, const int32_t *Tlen, float *gates, const float *Uf, const float *Ub,
                   const float *Pf, const float *Pb, float *hF, float *hB, float *cF, float *cB, const float *dh,
                   float *dz, unsigned int *counters, float *dc, const LstmZoneout *zo, cudaStream_t st) {
    LstmPlan p;
    const int ndir = Ub ? 2 : 1;
    const bool peep = (Pf != nullptr);
    const int rc = lstm_plan(H, B, ndir, peep, zo != nullptr, &p);
    if (rc != CTCB_OK) return rc;
    LstmZoArgs a;
    a.mode = mode; a.T = T; a.B = B; a.H = H; a.Tlen = Tlen; a.gates = gates;
    a.U[0] = Uf; a.U[1] = Ub ? Ub : Uf;
    a.h[0] = hF; a.h[1] = Ub ? hB : hF;
    a.c[0] = cF; a.c[1] = Ub ? cB : cF;
    a.dh = dh; a.dz = dz; a.dc = dc;
    a.ndir = ndir;
    a.P[0] = Pf; a.P[1] = Ub ? Pb : Pf;
    if (zo) {
        a.dhc = zo->dhc;
        a.train = zo->train ? 1 : 0;
        a.zc = zo->zc;
        a.zh = zo->zh;
        a.thr_c = zoneout_threshold(zo->zc);
        a.thr_h = zoneout_threshold(zo->zh);
        a.key = make_uint2((uint32_t)zo->seed, (uint32_t)(zo->seed >> 32));
        a.step = zo->step;
        a.first = zo->first;
        a.stride = zo->stride;
        a.layer = zo->layer;
    }
    const int slices = (H + LS_UNITS - 1) / LS_UNITS;
    return with_ki<2, 4, 8, 16, 32>(p.KI, [&](auto ki) {
        constexpr int KI = decltype(ki)::value;
        if (zo)
            return peep ? coop_launch(lstm_sweep_kernel<KI, true, true>, a, counters, slices, p.parts, p.smem, st)
                        : coop_launch(lstm_sweep_kernel<KI, false, true>, a, counters, slices, p.parts, p.smem, st);
        return peep ? coop_launch(lstm_sweep_kernel<KI, true, false>, static_cast<LstmPeepArgs &>(a), counters, slices,
                                  p.parts, p.smem, st)
                    : coop_launch(lstm_sweep_kernel<KI, false, false>, static_cast<LstmArgs &>(a), counters, slices,
                                  p.parts, p.smem, st);
    });
}

// ---- the peephole weight gradients -----------------------------------------------------------------------------
// dP_d[r][j] = sum over the rows (t, b) of dz_r[t][b][j] * c'[t][b][j], r = i, f, o (gate blocks 0, 1, 3 of direction
// d), c' = c_{t-1} (direction 0) / c_{t+1} (direction 1) for i and f, c_t for o; c' = 0 outside 0..T-1, and dz and c are
// 0 at the padded frames, so the sum needs no lengths.  Column q = (d, r, j) of ndir * 3H; stage 1 sums fixed chunks of
// LPG_ROWS rows per column (32 columns x 8 row lanes per CTA), stage 2 adds the chunks in order: the bits depend only
// on T, B, H and the inputs.
constexpr int LPG_ROWS = 1024;

__global__ void lstm_peephole_grad_stage1(const float *__restrict__ dz, const float *__restrict__ cF,
                                          const float *__restrict__ cB, int T, int B, int H, int ndir,
                                          float *__restrict__ partial) {
    __shared__ float sh[8][33];
    const int Q = ndir * 3 * H;
    const int q = blockIdx.x * 32 + threadIdx.x;
    const int64_t R = (int64_t)T * B;
    const int64_t r0 = (int64_t)blockIdx.y * LPG_ROWS;
    const int64_t r1 = (r0 + LPG_ROWS < R) ? r0 + LPG_ROWS : R;
    float s = 0.f;
    if (q < Q) {
        const int d = q / (3 * H), rr = (q - d * 3 * H) / H, j = q - d * 3 * H - rr * H;
        const int64_t G = (int64_t)ndir * 4 * H;
        const float *z = dz + (int64_t)d * 4 * H + (int64_t)(rr == 2 ? 3 : rr) * H + j;
        const float *c = (d == 0 ? cF : cB) + j;
        // the row of c' relative to the row of dz: the step before in this direction's order, or the frame itself
        const int64_t shift = (rr == 2) ? 0 : (d == 0 ? -(int64_t)B : (int64_t)B);
        for (int64_t r = r0 + threadIdx.y; r < r1; r += 8) {
            const int64_t rc = r + shift;
            const float cv = (rc >= 0 && rc < R) ? __ldg(c + rc * H) : 0.f;
            s = fmaf(__ldg(z + r * G), cv, s);
        }
    }
    sh[threadIdx.y][threadIdx.x] = s;
    __syncthreads();
    if (threadIdx.y == 0 && q < Q) {
        float t = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) t += sh[i][threadIdx.x];
        partial[(int64_t)blockIdx.y * Q + q] = t;
    }
}

template <bool ACC>
__global__ void lstm_peephole_grad_stage2(const float *__restrict__ partial, int nblk, int H, int ndir, float *dPf,
                                          float *dPb) {
    const int Q = ndir * 3 * H;
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= Q) return;
    float s = 0.f;
    for (int i = 0; i < nblk; ++i) s += partial[(int64_t)i * Q + q];
    float *out = (q < 3 * H) ? dPf + q : dPb + (q - 3 * H);
    if (ACC) s += *out;
    *out = s;
}

size_t lstm_peephole_grad_bytes(int64_t R, int H, int ndir) {
    const int64_t nblk = (R + LPG_ROWS - 1) / LPG_ROWS;
    return align_up((size_t)(nblk > 0 ? nblk : 1) * ndir * 3 * H * sizeof(float), 256);
}

// cB == nullptr: one direction (dz [T][B][4H]); partial: lstm_peephole_grad_bytes(T * B, H, ndir)
int run_lstm_peephole_grad(int T, int B, int H, const float *dz, const float *cF, const float *cB, float *dPf,
                           float *dPb, bool accumulate, float *partial, cudaStream_t st) {
    const int ndir = cB ? 2 : 1;
    const int Q = ndir * 3 * H;
    const int64_t R = (int64_t)T * B;
    const int nblk = (int)((R + LPG_ROWS - 1) / LPG_ROWS);
    lstm_peephole_grad_stage1<<<dim3((Q + 31) / 32, nblk), dim3(32, 8), 0, st>>>(dz, cF, cB ? cB : cF, T, B, H, ndir,
                                                                               partial);
    CTCB_LAUNCH_CHECK();
    if (accumulate) lstm_peephole_grad_stage2<true><<<(Q + 127) / 128, 128, 0, st>>>(partial, nblk, H, ndir, dPf, dPb);
    else lstm_peephole_grad_stage2<false><<<(Q + 127) / 128, 128, 0, st>>>(partial, nblk, H, ndir, dPf, dPb);
    CTCB_LAUNCH_CHECK();
    return CTCB_OK;
}

}  // namespace ctcb

extern "C" size_t ctcb_lstm_sweep_workspace_bytes(int H, int B) {
    if (H <= 0 || B <= 0) return 0;
    return 4096 + ctcb::lstm_carry_bytes(H, B);
}

extern "C" size_t ctcb_lstm_sweep_zoneout_workspace_bytes(int H, int B) {
    if (H <= 0 || B <= 0) return 0;
    return 4096 + 2 * ctcb::lstm_carry_bytes(H, B);
}

// zo non-null: the zoneout mode, whose dh carry follows the dc carry in scratch
static int lstm_sweep_entry(const char *name, int mode, int T, int B, int H, const int32_t *T_per_utt, float *gates,
                            const float *Uf, const float *Ub, const float *Pf, const float *Pb, float *hF, float *hB,
                            float *cF, float *cB, const float *dh, float *dz, ctcb::LstmZoneout *zo, void *scratch,
                            size_t scratch_bytes, void *stream) {
    using namespace ctcb;
    if (!T_per_utt || !gates || !Uf || !cF || !scratch || (mode == 0 && !hF) || (mode == 1 && (!dh || !dz)) ||
        (Ub && (!cB || (mode == 0 && !hB))))
        return set_error(CTCB_EINVAL, "%s: null pointer argument", name);
    if (T <= 0 || B <= 0 || H <= 0 || (mode != 0 && mode != 1))
        return set_error(CTCB_EINVAL, "%s: bad sizes", name);
    const size_t need = zo ? ctcb_lstm_sweep_zoneout_workspace_bytes(H, B) : ctcb_lstm_sweep_workspace_bytes(H, B);
    if (scratch_bytes < need || (((uintptr_t)scratch) & 255))
        return set_error(CTCB_ENOMEM, "%s: scratch of %zu bytes (256-byte aligned) needed, got %zu", name, need,
                         scratch_bytes);
    if (zo) zo->dhc = (float *)((char *)scratch + 4096 + lstm_carry_bytes(H, B));
    CTCB_CUDA_CHECK(cudaMemsetAsync(scratch, 0, 16 * sizeof(unsigned int), (cudaStream_t)stream));   // error flag
    return run_lstm_sweep(mode, T, B, H, T_per_utt, gates, Uf, Ub, Pf, Pb, hF, hB, cF, cB, dh, dz,
                          (unsigned int *)scratch, (float *)((char *)scratch + 4096), zo, (cudaStream_t)stream);
}

extern "C" int ctcb_lstm_sweep_f32(int mode, int T, int B, int H, const int32_t *T_per_utt, float *gates,
                                   const float *Uf, const float *Ub, float *hF, float *hB, float *cF, float *cB,
                                   const float *dh, float *dz, void *scratch, size_t scratch_bytes, void *stream) {
    return lstm_sweep_entry("ctcb_lstm_sweep_f32", mode, T, B, H, T_per_utt, gates, Uf, Ub, nullptr, nullptr, hF, hB,
                            cF, cB, dh, dz, nullptr, scratch, scratch_bytes, stream);
}

extern "C" int ctcb_lstm_sweep_peephole_f32(int mode, int T, int B, int H, const int32_t *T_per_utt, float *gates,
                                            const float *Uf, const float *Ub, const float *Pf, const float *Pb,
                                            float *hF, float *hB, float *cF, float *cB, const float *dh, float *dz,
                                            void *scratch, size_t scratch_bytes, void *stream) {
    if (!Pf || (Ub && !Pb)) return ctcb::set_error(CTCB_EINVAL, "ctcb_lstm_sweep_peephole_f32: null pointer argument");
    return lstm_sweep_entry("ctcb_lstm_sweep_peephole_f32", mode, T, B, H, T_per_utt, gates, Uf, Ub, Pf, Pb, hF, hB,
                            cF, cB, dh, dz, nullptr, scratch, scratch_bytes, stream);
}

extern "C" int ctcb_lstm_sweep_zoneout_f32(int mode, int T, int B, int H, const int32_t *T_per_utt, float *gates,
                                           const float *Uf, const float *Ub, const float *Pf, const float *Pb,
                                           float *hF, float *hB, float *cF, float *cB, const float *dh, float *dz,
                                           float zc, float zh, int train, uint64_t seed, const int64_t *step,
                                           int64_t first, int64_t stride, int layer, void *scratch,
                                           size_t scratch_bytes, void *stream) {
    using namespace ctcb;
    const char *name = "ctcb_lstm_sweep_zoneout_f32";
    if (Pf && Ub && !Pb) return set_error(CTCB_EINVAL, "%s: null pointer argument", name);
    if (!(zc >= 0.f && zc < 1.f) || !(zh >= 0.f && zh < 1.f))
        return set_error(CTCB_EINVAL, "%s: zc = %g, zh = %g (need both in [0, 1))", name, (double)zc, (double)zh);
    if (train && !step) return set_error(CTCB_EINVAL, "%s: training mode needs a step counter", name);
    if (first < 0 || stride < 1 || layer < 1 || layer > 255)
        return set_error(CTCB_EINVAL, "%s: first = %lld, stride = %lld, layer = %d (need first >= 0, stride >= 1, "
                         "1 <= layer <= 255)", name, (long long)first, (long long)stride, layer);
    LstmZoneout zo{zc, zh, train != 0, seed, step, first, stride, layer, nullptr};
    return lstm_sweep_entry(name, mode, T, B, H, T_per_utt, gates, Uf, Ub, Pf, Pf ? Pb : nullptr, hF, hB, cF, cB, dh,
                            dz, &zo, scratch, scratch_bytes, stream);
}

extern "C" size_t ctcb_lstm_peephole_grad_workspace_bytes(int T, int B, int H, int ndir) {
    if (T <= 0 || B <= 0 || H <= 0 || (ndir != 1 && ndir != 2)) return 0;
    return ctcb::lstm_peephole_grad_bytes((int64_t)T * B, H, ndir);
}

extern "C" int ctcb_lstm_peephole_grad_f32(int T, int B, int H, const float *dz, const float *cF, const float *cB,
                                           float *dPf, float *dPb, int accumulate, void *workspace, size_t ws_bytes,
                                           void *stream) {
    using namespace ctcb;
    if (!dz || !cF || !dPf || (cB && !dPb) || !workspace)
        return set_error(CTCB_EINVAL, "ctcb_lstm_peephole_grad_f32: null pointer argument");
    if (T <= 0 || B <= 0 || H <= 0 || (int64_t)T * B > 0x7fffffff)
        return set_error(CTCB_EINVAL, "ctcb_lstm_peephole_grad_f32: bad sizes (T=%d, B=%d, H=%d)", T, B, H);
    const size_t need = ctcb_lstm_peephole_grad_workspace_bytes(T, B, H, cB ? 2 : 1);
    if (ws_bytes < need)
        return set_error(CTCB_ENOMEM, "ctcb_lstm_peephole_grad_f32: workspace of %zu bytes needed, got %zu", need,
                         ws_bytes);
    return run_lstm_peephole_grad(T, B, H, dz, cF, cB, dPf, dPb, accumulate != 0, (float *)workspace,
                                  (cudaStream_t)stream);
}

static int debug_lstm_plan(int H, int B, int ndir, bool peep, bool zo, int32_t *out) {
    if (!out) return ctcb::set_error(CTCB_EINVAL, "ctcb_debug_lstm_plan: null output");
    ctcb::LstmPlan p;
    const int rc = ctcb::lstm_plan(H, B, ndir, peep, zo, &p);
    if (rc != CTCB_OK) return rc;
    out[0] = p.KI;
    out[1] = p.parts;
    out[2] = p.per_sm;
    out[3] = (ctcb::coop_tiles(B) + p.parts - 1) / p.parts;
    return CTCB_OK;
}

extern "C" int ctcb_debug_lstm_plan(int H, int B, int ndir, int peephole, int32_t *out) {
    return debug_lstm_plan(H, B, ndir, peephole != 0, false, out);
}

extern "C" int ctcb_debug_lstm_zoneout_plan(int H, int B, int ndir, int peephole, int32_t *out) {
    return debug_lstm_plan(H, B, ndir, peephole != 0, true, out);
}
