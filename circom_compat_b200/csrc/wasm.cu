// wasm.cu - circom 2 witness calculation on the device: a WebAssembly interpreter with one lane per witness.
//
// Host: b2g_wasm_load decodes and validates a module of the integer subset of WebAssembly 1.0 (MVP) and translates every
// function body into fixed-width instructions (Ins, 16 B).  Immediates are decoded, and every branch carries its target
// pc, the frame offset of the stack height it cuts back to and its result arity, so the device never reads LEB128 or
// walks blocks.  Validation types the operand stack, which gives each function's maximum height: a call checks once,
// on entry, that the callee's locals and operand stack fit in the lane's slots.
//
// Device: wasm_kernel runs one lane per witness.  Its linear memory, its operand stack + locals + globals ("slots") and
// its call frames sit in per-warp arrays where word i of lane l is next to word i of the warp's other lanes, so lanes
// running the same instruction make coalesced accesses.  Between the calls of the protocol the lane drives itself
// (driver_next): no host round trip.  Every memory access is checked against the lane's current memory size, every
// call against the slot and depth caps, and every instruction against the lane's fuel: a module can end a lane with a
// status, never fault the kernel or run without bound.
#include <algorithm>
#include <cstring>
#include <memory>
#include <string>
#include <vector>
#include "../../include/b2groth.h"
#include "fp.cuh"
#include "stage.cuh"
#include "util.cuh"
#include "verify.cuh"

namespace b2g {
namespace wasm {

constexpr uint32_t PAGE_WORDS = 16384;                // 64 KiB pages of 32-bit words
constexpr uint32_t EXIT_PC = 0xffffffffu;             // return address of a call made by the driver
constexpr uint32_t NO_FUNC = 0xffffffffu;             // empty table element
constexpr uint32_t MAX_GLOBALS = 1u << 20;            // globals sit in every lane's first slots
constexpr uint32_t MIN_SLOTS_ABOVE_GLOBALS = 8;       // the driver's call arguments and results sit right above them
// Default instruction budget per lane, sized for circuits of about a million constraints.  On an H100 (700 W) a lone lane
// ran 5.2 M instructions/s in a one-instruction loop and about 1.1 M/s on circuit2's code, so a lane stuck in a loop holds
// the call for roughly 14 to 65 minutes before it ends with B2G_WASM_FUEL; b2g_wasm_set_limits lowers it.
constexpr uint64_t DEFAULT_FUEL = 1ull << 32;

// lane statuses (b2groth.h B2G_WASM_*)
enum : uint32_t { ST_OK = 0, ST_UNREACHABLE = 1, ST_MEMORY = 2, ST_DIV_ZERO = 3, ST_OVERFLOW = 4, ST_STACK = 5,
                  ST_FUEL = 6, ST_INDIRECT = 7, ST_PROTOCOL = 8, ST_EXCEPTION = 0x100 };

// Internal opcodes.  Numeric, memory and constant instructions keep their WebAssembly opcode; control and variable
// access get their own, with every operand resolved by the translator.
enum : uint32_t {
    I_BR = 0x100,        // a target pc, b = frame offset of the height to cut back to, c arity
    I_BR_IF,             // the same when the popped i32 is not zero
    I_BR_UNLESS,         // a target pc when the popped i32 is zero (if)
    I_JMP,               // a target pc (else at the end of a then-arm)
    I_BR_TABLE,          // a entries follow (then the default), each an I_BR: the popped index picks one
    I_RETURN,            // c arity
    I_CALL,              // a function index (defined)
    I_CALL_HOST,         // a runtime import kind (0 exceptionHandler), b parameter count
    I_CALL_INDIRECT,     // a canonical type id
    I_LOCAL_GET, I_LOCAL_SET, I_LOCAL_TEE,   // a local index
    I_GLOBAL_GET, I_GLOBAL_SET,              // a global index (= slot)
    I_SELECT, I_DROP, I_UNREACHABLE,
    I_END_OP
};

struct Ins { uint32_t op, a, b, c; };
// entry pc (NO_FUNC for an import), parameters, locals with parameters, locals + max operand height, results, canonical
// type id, runtime import kind for an import, index in the type section
struct Fn { uint32_t entry, nparams, nlocals, frame, nresults, type_id, host_kind, type_index; };

// the per-call constants of the kernel
struct Prog {
    const Ins* code;
    const Fn* fns;
    const uint32_t* table; uint32_t table_size;
    const uint64_t* global_init; uint32_t nglobals;
    const uint32_t* image; uint32_t image_words;            // initial linear memory
    uint32_t init_pages, max_pages, slot_cap, depth_cap;
    uint64_t fuel;
    uint32_t* mem; uint64_t* slots; uint2* frames;          // per-warp interleaved lane state
    uint32_t lanes;                                          // lanes in this chunk
    int mode;                                                // 0 probe, 1 witness, 2 one exported call
    // protocol function indices: init, writeShared, setInput, getWitnessSize, getWitness, readShared, getVersion,
    // getFieldNumLen32, getRawPrime, getInputSize
    uint32_t fx[10];
    // witness: values (lane-major, n_values x 8 words each), the (msb, lsb, index) of each value, witness size
    const uint32_t* values; const uint3* value_meta; uint32_t n_values, n_wit, sanity;
    uint32_t* out;                                           // witness: lane-major n_wit x 8 words; probe: 16 words
    uint32_t* status;
    // mode 2: the export, its arguments (lane-major) and a result per lane
    uint32_t run_fn, run_nargs; const uint64_t* run_args; uint64_t* run_out;
};

enum { FX_INIT, FX_WRITE, FX_SET_INPUT, FX_WSIZE, FX_GETW, FX_READ, FX_VERSION, FX_N32, FX_PRIME, FX_ISIZE };

__device__ __forceinline__ uint32_t clz32(uint32_t x) { return __clz(x); }
__device__ __forceinline__ uint32_t ctz32(uint32_t x) { return __clz(__brev(x)); }
__device__ __forceinline__ uint64_t clz64(uint64_t x) { return __clzll(x); }
__device__ __forceinline__ uint64_t ctz64(uint64_t x) { return __clzll(__brevll(x)); }

struct Lane {
    uint32_t* mem; uint64_t* slot; uint2* frame;   // this lane's word 0; lane stride 32
    __device__ __forceinline__ uint32_t& mw(uint32_t i) const { return mem[(size_t)i * 32]; }
    __device__ __forceinline__ uint64_t& s(uint32_t i) const { return slot[(size_t)i * 32]; }
    __device__ __forceinline__ uint2& f(uint32_t i) const { return frame[(size_t)i * 32]; }
};

// n (1, 2, 4 or 8) bytes at byte address ea, already checked to lie inside the lane's memory
__device__ __forceinline__ uint64_t mem_read(const Lane& L, uint64_t ea, int n) {
    const uint32_t wi = (uint32_t)(ea >> 2), sh = (uint32_t)(ea & 3) * 8;
    if (sh == 0 && n == 4) return L.mw(wi);
    const uint32_t nw = ((uint32_t)(ea & 3) + n + 3) >> 2;
    uint64_t v = L.mw(wi);
    if (nw > 1) v |= (uint64_t)L.mw(wi + 1) << 32;
    uint64_t r = v >> sh;
    if (nw > 2) r |= (uint64_t)L.mw(wi + 2) << (64 - sh);
    return n == 8 ? r : r & ((1ull << (8 * n)) - 1);
}

__device__ __forceinline__ void mem_write(const Lane& L, uint64_t ea, int n, uint64_t v) {
    const uint32_t wi = (uint32_t)(ea >> 2), sh = (uint32_t)(ea & 3) * 8;
    if (sh == 0 && n == 4) { L.mw(wi) = (uint32_t)v; return; }
    if (sh == 0 && n == 8) { L.mw(wi) = (uint32_t)v; L.mw(wi + 1) = (uint32_t)(v >> 32); return; }
    const uint64_t mask = n == 8 ? ~0ull : (1ull << (8 * n)) - 1;
    const unsigned __int128 m = (unsigned __int128)mask << sh, x = (unsigned __int128)(v & mask) << sh;
    const uint32_t nw = ((uint32_t)(ea & 3) + n + 3) >> 2;
    for (uint32_t k = 0; k < nw; k++) {
        const uint32_t mk = (uint32_t)(m >> (32 * k)), xk = (uint32_t)(x >> (32 * k));
        L.mw(wi + k) = (L.mw(wi + k) & ~mk) | xk;
    }
}

__device__ __forceinline__ uint64_t sext(uint64_t v, int bits) {
    return (uint64_t)(((int64_t)(v << (64 - bits))) >> (64 - bits));
}

// The driver: after the lane's previous exported call returned (ret = its result, if any), picks the next call of the
// protocol and its arguments.  Returns false when the lane has finished.  seq counts the calls made so far.
__device__ __forceinline__ bool driver_next(const Prog& P, uint32_t lane, uint32_t seq, uint64_t ret, uint32_t& fn,
                                            uint64_t* args, uint32_t& nargs, uint32_t& status) {
    nargs = 0;
    if (P.mode == 2) {
        if (seq == 1) { if (P.fns[P.run_fn].nresults) P.run_out[lane] = ret; return false; }
        fn = P.run_fn; nargs = P.run_nargs;
        for (uint32_t k = 0; k < nargs; k++) args[k] = P.run_args[(size_t)lane * nargs + k];
        return true;
    }
    if (P.mode == 0) {   // getVersion, getFieldNumLen32, getRawPrime, readShared(0..7), getWitnessSize, getInputSize
        if (seq >= 1) {
            const uint32_t s = seq - 1;
            const int slot = s == 0 ? 0 : s == 1 ? 1 : s == 2 ? -1 : s < 11 ? (int)(s - 3) + 2 : (int)(s - 11) + 10;
            if (slot >= 0) P.out[slot] = (uint32_t)ret;
        }
        if (seq == 13) return false;
        if (seq == 0) fn = P.fx[FX_VERSION];
        else if (seq == 1) fn = P.fx[FX_N32];
        else if (seq == 2) fn = P.fx[FX_PRIME];
        else if (seq < 11) { fn = P.fx[FX_READ]; args[0] = seq - 3; nargs = 1; }
        else fn = seq == 11 ? P.fx[FX_WSIZE] : P.fx[FX_ISIZE];
        return true;
    }
    // witness: init(sanity); per value 8 x writeSharedRWMemory(j, limb) + setInputSignal(msb, lsb, i); getWitnessSize;
    // per witness getWitness(i) + 8 x readSharedRWMemory(j)
    const uint32_t nin = 9 * P.n_values, w0 = 2 + nin;
    if (seq == 0) { fn = P.fx[FX_INIT]; args[0] = P.sanity; nargs = 1; return true; }
    if (seq <= nin) {
        const uint32_t v = (seq - 1) / 9, j = (seq - 1) % 9;
        if (j < 8) {
            fn = P.fx[FX_WRITE]; args[0] = j; args[1] = P.values[((size_t)lane * P.n_values + v) * 8 + j]; nargs = 2;
        } else {
            const uint3 m = P.value_meta[v];
            fn = P.fx[FX_SET_INPUT]; args[0] = m.x; args[1] = m.y; args[2] = m.z; nargs = 3;
        }
        return true;
    }
    if (seq == nin + 1) { fn = P.fx[FX_WSIZE]; return true; }
    if (seq == w0 && (uint32_t)ret != P.n_wit) { status = ST_PROTOCOL; return false; }
    if (seq > w0) {                                 // the previous call was readSharedRWMemory(pj - 1) of witness pi
        const uint32_t pk = seq - 1 - w0, pi = pk / 9, pj = pk % 9;
        if (pj > 0) P.out[((size_t)lane * P.n_wit + pi) * 8 + (pj - 1)] = (uint32_t)ret;
    }
    const uint32_t k = seq - w0, i = k / 9, j = k % 9;
    if (i == P.n_wit) return false;
    if (j == 0) { fn = P.fx[FX_GETW]; args[0] = i; nargs = 1; }
    else { fn = P.fx[FX_READ]; args[0] = j - 1; nargs = 1; }
    return true;
}

__global__ void __launch_bounds__(128) wasm_kernel(const Prog P) {
    const uint32_t lane = blockIdx.x * blockDim.x + threadIdx.x;
    if (lane >= P.lanes) return;
    if ((uint64_t)P.nglobals + MIN_SLOTS_ABOVE_GLOBALS > P.slot_cap) { P.status[lane] = ST_STACK; return; }   // the host refuses this
    const uint32_t warp = lane >> 5, l = lane & 31;
    Lane L;
    L.mem = P.mem + (size_t)warp * P.max_pages * PAGE_WORDS * 32 + l;
    L.slot = P.slots + (size_t)warp * P.slot_cap * 32 + l;
    L.frame = P.frames + (size_t)warp * P.depth_cap * 32 + l;
    for (uint32_t i = 0; i < P.image_words; i++) L.mw(i) = __ldg(P.image + i);
    for (uint32_t g = 0; g < P.nglobals; g++) L.s(g) = __ldg(P.global_init + g);

    uint32_t pages = P.init_pages, status = ST_OK, seq = 0, depth = 0, pc = 0, fp = 0, sp = P.nglobals;
    uint64_t fuel = P.fuel, ret = 0;
    uint32_t fn; uint64_t args[3]; uint32_t nargs;

    // enters defined function f whose nparams arguments are the top of the stack; false (status set) if it does not fit
    auto enter = [&](uint32_t f, uint32_t ret_pc) -> bool {
        const Fn F = P.fns[f];
        const uint32_t nfp = sp - F.nparams;
        if (depth >= P.depth_cap || (uint64_t)nfp + F.frame > P.slot_cap) { status = ST_STACK; return false; }
        for (uint32_t k = F.nparams; k < F.nlocals; k++) L.s(nfp + k) = 0;
        L.f(depth) = make_uint2(ret_pc, fp);
        depth++;
        fp = nfp; sp = nfp + F.nlocals; pc = F.entry;
        return true;
    };
    // a call into the runtime imports: exceptionHandler ends the lane, the message functions are no-ops
    auto host = [&](uint32_t kind, uint32_t np) -> bool {
        if (kind == 0) { status = ST_EXCEPTION + (uint32_t)L.s(sp - 1); return false; }
        sp -= np;
        return true;
    };

    for (;;) {
        if (depth == 0) {                                  // the previous exported call returned (or none was made)
            if (seq > 0 && P.fns[fn].nresults) ret = L.s(P.nglobals);
            if (!driver_next(P, lane, seq, ret, fn, args, nargs, status)) break;
            seq++;
            sp = P.nglobals;
            for (uint32_t k = 0; k < nargs; k++) L.s(sp++) = args[k];
            const Fn F = P.fns[fn];
            if (F.entry == NO_FUNC) {                      // an export that is a runtime import
                if (!host(F.host_kind, F.nparams)) break;
                continue;
            }
            if (!enter(fn, EXIT_PC)) break;
        }
        if (fuel == 0) { status = ST_FUEL; break; }
        fuel--;
        const uint4 q = __ldg(reinterpret_cast<const uint4*>(P.code) + pc);
        const uint32_t op = q.x;
        pc++;
        bool ok = true;
        switch (op) {
            case I_LOCAL_GET: L.s(sp) = L.s(fp + q.y); sp++; break;
            case I_LOCAL_SET: sp--; L.s(fp + q.y) = L.s(sp); break;
            case I_LOCAL_TEE: L.s(fp + q.y) = L.s(sp - 1); break;
            case I_GLOBAL_GET: L.s(sp) = L.s(q.y); sp++; break;
            case I_GLOBAL_SET: sp--; L.s(q.y) = L.s(sp); break;
            case I_DROP: sp--; break;
            case I_SELECT: {
                const uint32_t c = (uint32_t)L.s(sp - 1);
                if (!c) L.s(sp - 3) = L.s(sp - 2);
                sp -= 2;
                break;
            }
            case I_UNREACHABLE: status = ST_UNREACHABLE; ok = false; break;
            case I_JMP: pc = q.y; break;
            case I_BR_UNLESS: sp--; if (!(uint32_t)L.s(sp)) pc = q.y; break;
            case I_BR_IF: sp--; if (!(uint32_t)L.s(sp)) break;
            [[fallthrough]];
            case I_BR: {
                const uint32_t dst = fp + q.z;
                for (uint32_t k = 0; k < q.w; k++) L.s(dst + k) = L.s(sp - q.w + k);
                sp = dst + q.w; pc = q.y;
                break;
            }
            case I_BR_TABLE: {
                sp--;
                const uint32_t i = (uint32_t)L.s(sp);
                const uint4 e = __ldg(reinterpret_cast<const uint4*>(P.code) + pc + min(i, q.y));
                const uint32_t dst = fp + e.z;
                for (uint32_t k = 0; k < e.w; k++) L.s(dst + k) = L.s(sp - e.w + k);
                sp = dst + e.w; pc = e.y;
                break;
            }
            case I_RETURN: {
                for (uint32_t k = 0; k < q.w; k++) L.s(fp + k) = L.s(sp - q.w + k);
                sp = fp + q.w;
                depth--;
                const uint2 fr = L.f(depth);
                pc = fr.x; fp = fr.y;
                break;
            }
            case I_CALL: ok = enter(q.y, pc); break;
            case I_CALL_HOST: ok = host(q.y, q.z); break;
            case I_CALL_INDIRECT: {
                sp--;
                const uint32_t i = (uint32_t)L.s(sp);
                const uint32_t f = i < P.table_size ? P.table[i] : NO_FUNC;
                if (f == NO_FUNC || P.fns[f].type_id != q.y) { status = ST_INDIRECT; ok = false; break; }
                const Fn F = P.fns[f];
                ok = F.entry == NO_FUNC ? host(F.host_kind, F.nparams) : enter(f, pc);
                break;
            }
            case 0x41: L.s(sp) = q.y; sp++; break;                                  // i32.const
            case 0x42: L.s(sp) = ((uint64_t)q.z << 32) | q.y; sp++; break;          // i64.const
            case 0x3f: L.s(sp) = pages; sp++; break;                                // memory.size
            case 0x40: {                                                            // memory.grow
                const uint32_t d = (uint32_t)L.s(sp - 1);
                if ((uint64_t)pages + d > P.max_pages) { L.s(sp - 1) = 0xffffffffu; break; }
                for (uint32_t i = pages * PAGE_WORDS; i < (pages + d) * PAGE_WORDS; i++) L.mw(i) = 0;
                L.s(sp - 1) = pages;
                pages += d;
                break;
            }
            default:
                if (op >= 0x28 && op <= 0x3e) {                                     // loads and stores
                    const bool store = op >= 0x36;
                    int n; bool sg = false, w64 = false;
                    switch (op) {
                        case 0x28: n = 4; break;              case 0x29: n = 8; w64 = true; break;
                        case 0x2c: n = 1; sg = true; break;   case 0x2d: n = 1; break;
                        case 0x2e: n = 2; sg = true; break;   case 0x2f: n = 2; break;
                        case 0x30: n = 1; sg = w64 = true; break; case 0x31: n = 1; w64 = true; break;
                        case 0x32: n = 2; sg = w64 = true; break; case 0x33: n = 2; w64 = true; break;
                        case 0x34: n = 4; sg = w64 = true; break; case 0x35: n = 4; w64 = true; break;
                        case 0x36: n = 4; break; case 0x37: n = 8; break; case 0x3a: n = 1; break; case 0x3b: n = 2; break;
                        case 0x3c: n = 1; break; case 0x3d: n = 2; break; default: n = 4; break;   // 0x3e
                    }
                    const uint32_t ai = store ? sp - 2 : sp - 1;
                    const uint64_t ea = (uint64_t)(uint32_t)L.s(ai) + q.y;
                    if (ea + n > (uint64_t)pages * PAGE_WORDS * 4) { status = ST_MEMORY; ok = false; break; }
                    if (store) {
                        mem_write(L, ea, n, L.s(sp - 1));
                        sp -= 2;
                    } else {
                        uint64_t v = mem_read(L, ea, n);
                        if (sg) v = sext(v, 8 * n);
                        L.s(ai) = w64 ? v : (uint64_t)(uint32_t)v;
                    }
                    break;
                }
                if ((op >= 0x45 && op <= 0x4f) || (op >= 0x67 && op <= 0x78) || op == 0xc0 || op == 0xc1) {   // i32
                    const bool unary = op == 0x45 || (op >= 0x67 && op <= 0x69) || op >= 0xc0;
                    const uint32_t a = (uint32_t)L.s(unary ? sp - 1 : sp - 2), b = unary ? 0 : (uint32_t)L.s(sp - 1);
                    const int32_t sa = (int32_t)a, sb = (int32_t)b;
                    uint32_t r = 0;
                    switch (op) {
                        case 0x45: r = a == 0; break;
                        case 0x46: r = a == b; break; case 0x47: r = a != b; break;
                        case 0x48: r = sa < sb; break; case 0x49: r = a < b; break;
                        case 0x4a: r = sa > sb; break; case 0x4b: r = a > b; break;
                        case 0x4c: r = sa <= sb; break; case 0x4d: r = a <= b; break;
                        case 0x4e: r = sa >= sb; break; case 0x4f: r = a >= b; break;
                        case 0x67: r = clz32(a); break; case 0x68: r = ctz32(a); break; case 0x69: r = __popc(a); break;
                        case 0x6a: r = a + b; break; case 0x6b: r = a - b; break; case 0x6c: r = a * b; break;
                        case 0x6d:
                            if (b == 0) { status = ST_DIV_ZERO; ok = false; break; }
                            if (sa == INT32_MIN && sb == -1) { status = ST_OVERFLOW; ok = false; break; }
                            r = (uint32_t)(sa / sb); break;
                        case 0x6e: if (b == 0) { status = ST_DIV_ZERO; ok = false; break; } r = a / b; break;
                        case 0x6f:
                            if (b == 0) { status = ST_DIV_ZERO; ok = false; break; }
                            r = sb == -1 ? 0 : (uint32_t)(sa % sb); break;
                        case 0x70: if (b == 0) { status = ST_DIV_ZERO; ok = false; break; } r = a % b; break;
                        case 0x71: r = a & b; break; case 0x72: r = a | b; break; case 0x73: r = a ^ b; break;
                        case 0x74: r = a << (b & 31); break;
                        case 0x75: r = (uint32_t)(sa >> (b & 31)); break;
                        case 0x76: r = a >> (b & 31); break;
                        case 0x77: r = (a << (b & 31)) | (a >> ((32 - (b & 31)) & 31)); break;
                        case 0x78: r = (a >> (b & 31)) | (a << ((32 - (b & 31)) & 31)); break;
                        case 0xc0: r = (uint32_t)(int32_t)(int8_t)a; break;
                        default: r = (uint32_t)(int32_t)(int16_t)a; break;   // 0xc1
                    }
                    if (!ok) break;
                    if (!unary) sp--;
                    L.s(sp - 1) = r;
                    break;
                }
                {                                                                   // i64 and conversions
                    const bool unary = op == 0x50 || (op >= 0x79 && op <= 0x7b) || op == 0xa7 || op == 0xac ||
                                       op == 0xad || op >= 0xc2;
                    const uint64_t a = L.s(unary ? sp - 1 : sp - 2), b = unary ? 0 : L.s(sp - 1);
                    const int64_t sa = (int64_t)a, sb = (int64_t)b;
                    uint64_t r = 0;
                    switch (op) {
                        case 0x50: r = a == 0; break;
                        case 0x51: r = a == b; break; case 0x52: r = a != b; break;
                        case 0x53: r = sa < sb; break; case 0x54: r = a < b; break;
                        case 0x55: r = sa > sb; break; case 0x56: r = a > b; break;
                        case 0x57: r = sa <= sb; break; case 0x58: r = a <= b; break;
                        case 0x59: r = sa >= sb; break; case 0x5a: r = a >= b; break;
                        case 0x79: r = clz64(a); break; case 0x7a: r = ctz64(a); break; case 0x7b: r = __popcll(a); break;
                        case 0x7c: r = a + b; break; case 0x7d: r = a - b; break; case 0x7e: r = a * b; break;
                        case 0x7f:
                            if (b == 0) { status = ST_DIV_ZERO; ok = false; break; }
                            if (sa == INT64_MIN && sb == -1) { status = ST_OVERFLOW; ok = false; break; }
                            r = (uint64_t)(sa / sb); break;
                        case 0x80: if (b == 0) { status = ST_DIV_ZERO; ok = false; break; } r = a / b; break;
                        case 0x81:
                            if (b == 0) { status = ST_DIV_ZERO; ok = false; break; }
                            r = sb == -1 ? 0 : (uint64_t)(sa % sb); break;
                        case 0x82: if (b == 0) { status = ST_DIV_ZERO; ok = false; break; } r = a % b; break;
                        case 0x83: r = a & b; break; case 0x84: r = a | b; break; case 0x85: r = a ^ b; break;
                        case 0x86: r = a << (b & 63); break;
                        case 0x87: r = (uint64_t)(sa >> (b & 63)); break;
                        case 0x88: r = a >> (b & 63); break;
                        case 0x89: r = (a << (b & 63)) | (a >> ((64 - (b & 63)) & 63)); break;
                        case 0x8a: r = (a >> (b & 63)) | (a << ((64 - (b & 63)) & 63)); break;
                        case 0xa7: r = (uint32_t)a; break;
                        case 0xac: r = (uint64_t)(int64_t)(int32_t)(uint32_t)a; break;
                        case 0xad: r = (uint32_t)a; break;
                        case 0xc2: r = sext(a, 8); break; case 0xc3: r = sext(a, 16); break;
                        default: r = sext(a, 32); break;   // 0xc4
                    }
                    if (!ok) break;
                    if (!unary) sp--;
                    L.s(sp - 1) = r;
                }
                break;
        }
        if (!ok) break;
    }
    P.status[lane] = status;
}

// canonical words (lane-major, n per lane) -> Montgomery, in place
__global__ void wasm_to_mont_kernel(uint32_t* w, size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    fe a = fe_load(w + 8 * i);
    fe_store(w + 8 * i, Fr::from_canonical(a));
}

}  // namespace wasm
}  // namespace b2g

// ================================================================================================================ host
using namespace b2g;
using namespace b2g::wasm;

namespace {

[[noreturn]] void refuse(const std::string& m) { throw_error(B2G_E_SHAPE, "wasm: " + m); }

const char* const RUNTIME_IMPORTS[4] = {"exceptionHandler", "printErrorMessage", "writeBufferMessage", "showSharedRWMemory"};
const uint32_t RUNTIME_PARAMS[4] = {1, 0, 0, 0};
// in the order of Prog::fx
const char* const PROTOCOL[10] = {"init", "writeSharedRWMemory", "setInputSignal", "getWitnessSize", "getWitness",
                                  "readSharedRWMemory", "getVersion", "getFieldNumLen32", "getRawPrime", "getInputSize"};
const uint8_t T_I32 = 0x7f, T_I64 = 0x7e, T_ANY = 0;

struct Reader {
    const uint8_t* b; size_t p, end;
    uint8_t byte() { if (p >= end) refuse("truncated module"); return b[p++]; }
    uint64_t uleb(int bits = 32) {
        uint64_t r = 0; int s = 0;
        for (;;) {
            const uint8_t v = byte();
            if (s > 63) refuse("malformed LEB128 integer");
            r |= (uint64_t)(v & 0x7f) << s; s += 7;
            if (!(v & 0x80)) break;
        }
        if (bits < 64 && (r >> bits)) refuse("LEB128 integer out of range");
        return r;
    }
    uint64_t sleb(int bits) {
        uint64_t r = 0; int s = 0; uint8_t v;
        do {
            v = byte();
            if (s >= 70) refuse("malformed LEB128 integer");
            if (s < 64) r |= (uint64_t)(v & 0x7f) << s;
            s += 7;
        } while (v & 0x80);
        if (s < 64 && (v & 0x40)) r |= ~0ull << s;
        return bits == 32 ? (uint64_t)(uint32_t)r : r;
    }
    std::string name() {
        const uint32_t n = (uint32_t)uleb();
        if (end - p < n) refuse("truncated name");
        std::string s((const char*)b + p, n); p += n; return s;
    }
};

struct FuncType { std::vector<uint8_t> params, results; };
struct Global { uint8_t type, mut; uint64_t init; };

struct Ctl {
    uint8_t kind;                 // 0 block, 1 loop, 2 if, 3 function
    uint8_t type;                 // result type, 0 for none
    uint32_t height, start;       // operand height at entry, pc of a loop's start
    bool unreachable = false, has_else = false;
    uint32_t if_fix = 0;          // pc of an if's I_BR_UNLESS until its else or end
    std::vector<uint32_t> fix;    // instructions that branch to the end
};

}  // namespace

struct b2g_wasm {
    int device = 0;
    bool circom = false;
    std::vector<FuncType> types;
    std::vector<uint32_t> type_id;                 // canonical id of each type (equal signatures, equal ids)
    std::vector<Fn> fns;
    std::vector<Ins> code;
    std::vector<uint32_t> table, image;
    std::vector<Global> globals;
    std::vector<std::pair<std::string, uint32_t>> exports;   // exported functions
    uint32_t nimports = 0, init_pages = 0, decl_max_pages = 65536;
    uint32_t fx[10] = {};
    b2g_wasm_summary info = {};
    b2g_wasm_limits lim = {};
    Ins* d_code = nullptr; Fn* d_fns = nullptr; uint32_t *d_table = nullptr, *d_image = nullptr; uint64_t* d_glob = nullptr;
    ~b2g_wasm() {
        cudaFree(d_code); cudaFree(d_fns); cudaFree(d_table); cudaFree(d_image); cudaFree(d_glob);
    }
    int find_export(const std::string& n) const {
        for (auto& e : exports) if (e.first == n) return (int)e.second;
        return -1;
    }
};

namespace {

uint64_t const_expr(Reader& r, const std::vector<Global>& globals, uint8_t want) {
    const uint8_t op = r.byte();
    uint64_t v; uint8_t t;
    if (op == 0x41) { v = r.sleb(32); t = T_I32; }
    else if (op == 0x42) { v = r.sleb(64); t = T_I64; }
    else if (op == 0x23) {
        const uint32_t g = (uint32_t)r.uleb();
        if (g >= globals.size()) refuse("constant expression reads an unknown global");
        v = globals[g].init; t = globals[g].type;
    } else refuse("constant expression opcode 0x" + [&] { char b[8]; snprintf(b, 8, "%02x", op); return std::string(b); }());
    if (r.byte() != 0x0b) refuse("constant expression is not a single constant");
    if (want && t != want) refuse("constant expression of the wrong type");
    return v;
}

std::string hex2(uint32_t op) { char b[16]; snprintf(b, sizeof b, "0x%02x", op); return b; }

// Translates and validates the body of defined function fi (whole index) into w->code.
void translate(b2g_wasm* w, uint32_t fi, Reader r, const FuncType& ft, uint32_t nparams) {
    std::vector<uint8_t> locals(ft.params.begin(), ft.params.end());
    const uint32_t ngroups = (uint32_t)r.uleb();
    for (uint32_t g = 0; g < ngroups; g++) {
        const uint32_t n = (uint32_t)r.uleb();
        const uint8_t t = r.byte();
        if (t != T_I32 && t != T_I64) refuse("function " + std::to_string(fi) + ": local of value type " + hex2(t) + " is not supported");
        if (locals.size() + n > 50000) refuse("function " + std::to_string(fi) + ": too many locals");
        locals.insert(locals.end(), n, t);
    }
    const uint32_t nloc = (uint32_t)locals.size();
    Fn& F = w->fns[fi];
    F.entry = (uint32_t)w->code.size(); F.nparams = nparams; F.nlocals = nloc;
    F.nresults = (uint32_t)ft.results.size();
    std::vector<uint8_t> vt;              // operand types
    uint32_t maxh = 0;
    std::vector<Ctl> ctl;
    Ctl top; top.kind = 3; top.type = ft.results.empty() ? 0 : ft.results[0]; top.height = 0; top.start = 0;
    ctl.push_back(top);
    auto& code = w->code;
    const std::string where = "function " + std::to_string(fi);
    auto bad = [&](const std::string& m) { refuse(where + ": " + m); };
    auto push = [&](uint8_t t) { vt.push_back(t); maxh = std::max<uint32_t>(maxh, (uint32_t)vt.size()); };
    auto pop = [&](uint8_t want) -> uint8_t {
        Ctl& c = ctl.back();
        if (vt.size() == c.height) {
            if (c.unreachable) return want;
            bad("operand stack underflow");
        }
        const uint8_t t = vt.back(); vt.pop_back();
        if (want != T_ANY && t != T_ANY && t != want) bad("operand type mismatch");
        return t;
    };
    auto emit = [&](uint32_t op, uint32_t a = 0, uint32_t b = 0, uint32_t c = 0) { code.push_back({op, a, b, c}); return (uint32_t)code.size() - 1; };
    auto set_unreachable = [&] { Ctl& c = ctl.back(); vt.resize(c.height); c.unreachable = true; };
    auto label_arity = [&](const Ctl& c) -> uint32_t { return c.kind == 1 ? 0 : (c.type ? 1 : 0); };
    // a branch instruction to relative depth d: fills target (or a fixup), height and arity; checks the label's values
    auto branch = [&](uint32_t op, uint32_t d) {
        if (d >= ctl.size()) bad("branch depth out of range");
        Ctl& c = ctl[ctl.size() - 1 - d];
        const uint32_t ar = label_arity(c);
        if (ar) { const uint8_t t = pop(c.type); push(t); }
        const uint32_t at = emit(op, 0, nloc + c.height, ar);
        if (c.kind == 1) code[at].a = c.start; else c.fix.push_back(at);
        return at;
    };
    auto mem_check = [&](uint32_t natural) -> uint32_t {
        const uint32_t align = (uint32_t)r.uleb();
        const uint32_t off = (uint32_t)r.uleb();
        if ((1u << std::min<uint32_t>(align, 31)) > natural) bad("alignment larger than natural");
        if (w->init_pages == 0 && w->decl_max_pages == 0) bad("memory access without a memory");
        return off;
    };

    while (!ctl.empty()) {
        const uint8_t op = r.byte();
        switch (op) {
            case 0x00: emit(I_UNREACHABLE); set_unreachable(); break;
            case 0x01: break;
            case 0x02: case 0x03: case 0x04: {
                const uint8_t bt = r.byte();
                if (bt != 0x40 && bt != T_I32 && bt != T_I64) bad("block type " + hex2(bt) + " is not supported");
                if (op == 0x04) pop(T_I32);
                Ctl c; c.kind = op == 0x02 ? 0 : op == 0x03 ? 1 : 2; c.type = bt == 0x40 ? 0 : bt;
                c.height = (uint32_t)vt.size(); c.start = (uint32_t)code.size();
                if (op == 0x04) c.if_fix = emit(I_BR_UNLESS);
                ctl.push_back(std::move(c));
                break;
            }
            case 0x05: {
                Ctl& c = ctl.back();
                if (c.kind != 2 || c.has_else) bad("else without if");
                if (c.type) pop(c.type);
                if (vt.size() != c.height) bad("values left on the stack at else");
                c.fix.push_back(emit(I_JMP));
                code[c.if_fix].a = (uint32_t)code.size();
                c.has_else = true; c.unreachable = false;
                break;
            }
            case 0x0b: {
                Ctl c = std::move(ctl.back());
                if (c.type) pop(c.type);
                if (vt.size() != c.height) bad("values left on the stack at end");
                if (c.kind == 2 && !c.has_else) {
                    if (c.type) bad("if with a result and no else");
                    code[c.if_fix].a = (uint32_t)code.size();
                }
                ctl.pop_back();
                if (c.kind == 3) {
                    const uint32_t at = emit(I_RETURN, 0, 0, c.type ? 1 : 0);
                    for (uint32_t f : c.fix) code[f].a = at;
                } else {
                    for (uint32_t f : c.fix) code[f].a = (uint32_t)code.size();
                    if (c.type) push(c.type);
                }
                break;
            }
            case 0x0c: branch(I_BR, (uint32_t)r.uleb()); set_unreachable(); break;
            case 0x0d: pop(T_I32); branch(I_BR_IF, (uint32_t)r.uleb()); break;
            case 0x0e: {
                const uint32_t n = (uint32_t)r.uleb();
                if (n > 1000000) bad("br_table too large");
                pop(T_I32);
                emit(I_BR_TABLE, n);
                int ar = -1;
                for (uint32_t k = 0; k <= n; k++) {
                    const uint32_t d = (uint32_t)r.uleb();
                    if (d >= ctl.size()) bad("branch depth out of range");
                    const uint32_t a = label_arity(ctl[ctl.size() - 1 - d]);
                    if (ar >= 0 && (uint32_t)ar != a) bad("br_table targets of different arity");
                    ar = (int)a;
                    branch(I_BR, d);
                }
                set_unreachable();
                break;
            }
            case 0x0f: {
                if (top.type) { const uint8_t t = pop(top.type); push(t); }
                emit(I_RETURN, 0, 0, top.type ? 1 : 0);
                set_unreachable();
                break;
            }
            case 0x10: case 0x11: {
                uint32_t tidx;
                if (op == 0x10) {
                    const uint32_t f = (uint32_t)r.uleb();
                    if (f >= w->fns.size()) bad("call of an unknown function");
                    tidx = w->fns[f].type_index;
                    if (f < w->nimports) emit(I_CALL_HOST, w->fns[f].host_kind, w->fns[f].nparams);
                    else emit(I_CALL, f);
                } else {
                    tidx = (uint32_t)r.uleb();
                    if (r.byte() != 0) bad("call_indirect on a table other than 0");
                    if (tidx >= w->types.size()) bad("call_indirect of an unknown type");
                    if (w->table.empty()) bad("call_indirect without a table");
                    pop(T_I32);
                    emit(I_CALL_INDIRECT, w->type_id[tidx]);
                }
                const FuncType& t = w->types[tidx];
                for (size_t k = t.params.size(); k-- > 0;) pop(t.params[k]);
                for (uint8_t x : t.results) push(x);
                // the callee's arguments occupy the caller's stack until it returns; room for its results too
                break;
            }
            case 0x1a: pop(T_ANY); emit(I_DROP); break;
            case 0x1b: {
                pop(T_I32);
                const uint8_t b = pop(T_ANY), a = pop(b);
                push(a != T_ANY ? a : b);
                emit(I_SELECT);
                break;
            }
            case 0x20: case 0x21: case 0x22: {
                const uint32_t x = (uint32_t)r.uleb();
                if (x >= nloc) bad("unknown local " + std::to_string(x));
                if (op == 0x20) push(locals[x]);
                else { pop(locals[x]); if (op == 0x22) push(locals[x]); }
                emit(op == 0x20 ? I_LOCAL_GET : op == 0x21 ? I_LOCAL_SET : I_LOCAL_TEE, x);
                break;
            }
            case 0x23: case 0x24: {
                const uint32_t x = (uint32_t)r.uleb();
                if (x >= w->globals.size()) bad("unknown global " + std::to_string(x));
                if (op == 0x23) push(w->globals[x].type);
                else { if (!w->globals[x].mut) bad("global.set of an immutable global"); pop(w->globals[x].type); }
                emit(op == 0x23 ? I_GLOBAL_GET : I_GLOBAL_SET, x);
                break;
            }
            case 0x28: case 0x29: case 0x2c: case 0x2d: case 0x2e: case 0x2f: case 0x30: case 0x31: case 0x32: case 0x33:
            case 0x34: case 0x35: {
                static const uint8_t nat[14] = {4, 8, 0, 0, 1, 1, 2, 2, 1, 1, 2, 2, 4, 4};
                const uint32_t off = mem_check(nat[op - 0x28]);
                pop(T_I32);
                push(op == 0x28 || (op >= 0x2c && op <= 0x2f) ? T_I32 : T_I64);
                emit(op, off);
                break;
            }
            case 0x36: case 0x37: case 0x3a: case 0x3b: case 0x3c: case 0x3d: case 0x3e: {
                static const uint8_t nat[9] = {4, 8, 0, 0, 1, 2, 1, 2, 4};
                const uint32_t off = mem_check(nat[op - 0x36]);
                pop(op == 0x36 || op == 0x3a || op == 0x3b ? T_I32 : T_I64);
                pop(T_I32);
                emit(op, off);
                break;
            }
            case 0x3f: case 0x40:
                if (r.byte() != 0) bad("memory index other than 0");
                if (op == 0x40) pop(T_I32);
                push(T_I32); emit(op);
                break;
            case 0x41: { const uint64_t v = r.sleb(32); push(T_I32); emit(op, (uint32_t)v); break; }
            case 0x42: { const uint64_t v = r.sleb(64); push(T_I64); emit(op, (uint32_t)v, (uint32_t)(v >> 32)); break; }
            default: {
                uint8_t in1, in2 = 0, out;     // in2 = 0: unary
                if (op == 0x45 || op == 0x67 || op == 0x68 || op == 0x69 || op == 0xc0 || op == 0xc1) { in1 = T_I32; out = T_I32; }
                else if (op >= 0x46 && op <= 0x4f) { in1 = in2 = T_I32; out = T_I32; }
                else if (op == 0x50) { in1 = T_I64; out = T_I32; }
                else if (op >= 0x51 && op <= 0x5a) { in1 = in2 = T_I64; out = T_I32; }
                else if (op >= 0x6a && op <= 0x78) { in1 = in2 = T_I32; out = T_I32; }
                else if ((op >= 0x79 && op <= 0x7b) || (op >= 0xc2 && op <= 0xc4)) { in1 = T_I64; out = T_I64; }
                else if (op >= 0x7c && op <= 0x8a) { in1 = in2 = T_I64; out = T_I64; }
                else if (op == 0xa7) { in1 = T_I64; out = T_I32; }
                else if (op == 0xac || op == 0xad) { in1 = T_I32; out = T_I64; }
                else bad("opcode " + hex2(op) + " is not in the integer subset of WebAssembly 1.0");
                if (in2) pop(in2);
                pop(in1);
                push(out);
                emit(op);
            }
        }
    }
    if (r.p != r.end) refuse(where + ": code after the end of the body");
    F.frame = nloc + maxh;
}

void load_module(b2g_wasm* w, const uint8_t* data, size_t len) {
    if (len < 8 || memcmp(data, "\0asm", 4) != 0) refuse("not a WebAssembly binary (no \\0asm magic)");
    if (memcmp(data + 4, "\x01\0\0\0", 4) != 0) refuse("WebAssembly binary version other than 1");
    Reader r{data, 8, len};
    std::vector<uint32_t> func_types;
    std::vector<std::pair<size_t, size_t>> bodies;
    bool have_mem = false;
    uint32_t table_min = 0; bool have_table = false;
    struct Seg { uint32_t off; size_t p, n; };
    std::vector<Seg> datas;
    std::vector<std::pair<uint32_t, std::vector<uint32_t>>> elems;
    int last_id = 0;
    while (r.p < len) {
        const uint8_t id = r.byte();
        const uint32_t size = (uint32_t)r.uleb();
        if (len - r.p < size) refuse("section runs past the end of the module");
        Reader s{data, r.p, r.p + size};
        r.p += size;
        if (id != 0) {
            if (id <= last_id) refuse("sections out of order");
            last_id = id;
        }
        switch (id) {
            case 0: break;   // custom
            case 1: {
                const uint32_t n = (uint32_t)s.uleb();
                for (uint32_t i = 0; i < n; i++) {
                    if (s.byte() != 0x60) refuse("malformed function type");
                    FuncType t;
                    for (int side = 0; side < 2; side++) {
                        const uint32_t k = (uint32_t)s.uleb();
                        for (uint32_t j = 0; j < k; j++) {
                            const uint8_t v = s.byte();
                            if (v != T_I32 && v != T_I64) refuse("function type " + std::to_string(i) + " has value type " + hex2(v) + ", which is not supported");
                            (side ? t.results : t.params).push_back(v);
                        }
                    }
                    if (t.results.size() > 1) refuse("function type " + std::to_string(i) + " has several results (multi-value)");
                    uint32_t id2 = (uint32_t)w->types.size();
                    for (size_t j = 0; j < w->types.size(); j++)
                        if (w->types[j].params == t.params && w->types[j].results == t.results) { id2 = w->type_id[j]; break; }
                    w->types.push_back(t); w->type_id.push_back(id2);
                }
                break;
            }
            case 2: {
                const uint32_t n = (uint32_t)s.uleb();
                for (uint32_t i = 0; i < n; i++) {
                    const std::string mod = s.name(), nm = s.name();
                    const uint8_t kind = s.byte();
                    if (kind != 0)
                        refuse("import " + mod + "." + nm + " is not a function" +
                               (mod == "env" && nm == "memory" ? " (a circom 1 module: it imports env.memory; only circom 2 modules are supported)" : ""));
                    int k = -1;
                    for (int j = 0; j < 4; j++) if (mod == "runtime" && nm == RUNTIME_IMPORTS[j]) k = j;
                    if (k < 0) refuse("import " + mod + "." + nm + " is not one of the circom 2 runtime functions");
                    const uint32_t t = (uint32_t)s.uleb();
                    if (t >= w->types.size()) refuse("import of an unknown type");
                    if (w->types[t].params.size() != RUNTIME_PARAMS[k] || !w->types[t].results.empty() ||
                        (k == 0 && w->types[t].params[0] != T_I32))
                        refuse("import runtime." + nm + " has the wrong signature");
                    Fn f = {NO_FUNC, RUNTIME_PARAMS[k], 0, 0, 0, w->type_id[t], (uint32_t)k, t};
                    w->fns.push_back(f);
                }
                w->nimports = (uint32_t)w->fns.size();
                break;
            }
            case 3: {
                const uint32_t n = (uint32_t)s.uleb();
                for (uint32_t i = 0; i < n; i++) {
                    const uint32_t t = (uint32_t)s.uleb();
                    if (t >= w->types.size()) refuse("function of an unknown type");
                    func_types.push_back(t);
                    const FuncType& ft = w->types[t];
                    Fn f = {0, (uint32_t)ft.params.size(), 0, 0, (uint32_t)ft.results.size(), w->type_id[t], 0, t};
                    w->fns.push_back(f);
                }
                break;
            }
            case 4: {
                const uint32_t n = (uint32_t)s.uleb();
                if (n > 1) refuse("more than one table");
                if (n) {
                    if (s.byte() != 0x70) refuse("table of a type other than funcref");
                    const uint8_t fl = s.byte();
                    table_min = (uint32_t)s.uleb();
                    if (fl & 1) s.uleb();
                    if (table_min > (1u << 20)) refuse("table too large");
                    have_table = true;
                }
                break;
            }
            case 5: {
                const uint32_t n = (uint32_t)s.uleb();
                if (n > 1) refuse("more than one memory");
                if (n) {
                    const uint8_t fl = s.byte();
                    w->init_pages = (uint32_t)s.uleb();
                    w->decl_max_pages = (fl & 1) ? (uint32_t)s.uleb() : 65536;
                    if (w->init_pages > 65536 || w->decl_max_pages > 65536 || w->decl_max_pages < w->init_pages) refuse("bad memory limits");
                    have_mem = true;
                }
                break;
            }
            case 6: {
                const uint32_t n = (uint32_t)s.uleb();
                if (n > MAX_GLOBALS) refuse("the module has " + std::to_string(n) + " globals; at most " + std::to_string(MAX_GLOBALS) + " are supported");
                for (uint32_t i = 0; i < n; i++) {
                    Global g;
                    g.type = s.byte(); g.mut = s.byte();
                    if (g.type != T_I32 && g.type != T_I64) refuse("global " + std::to_string(i) + " of value type " + hex2(g.type) + " is not supported");
                    g.init = const_expr(s, w->globals, g.type);
                    w->globals.push_back(g);
                }
                break;
            }
            case 7: {
                const uint32_t n = (uint32_t)s.uleb();
                for (uint32_t i = 0; i < n; i++) {
                    const std::string nm = s.name();
                    const uint8_t kind = s.byte();
                    const uint32_t idx = (uint32_t)s.uleb();
                    if (kind == 0) {
                        if (idx >= w->fns.size()) refuse("export of an unknown function");
                        w->exports.push_back({nm, idx});
                    }
                }
                break;
            }
            case 8: refuse("a start function is not supported");
            case 9: {
                const uint32_t n = (uint32_t)s.uleb();
                for (uint32_t i = 0; i < n; i++) {
                    if (s.uleb() != 0) refuse("element segment other than an active segment of table 0");
                    const uint32_t off = (uint32_t)const_expr(s, w->globals, T_I32);
                    const uint32_t k = (uint32_t)s.uleb();
                    std::vector<uint32_t> fs;
                    for (uint32_t j = 0; j < k; j++) {
                        const uint32_t f = (uint32_t)s.uleb();
                        if (f >= w->fns.size()) refuse("element of an unknown function");
                        fs.push_back(f);
                    }
                    elems.push_back({off, fs});
                }
                break;
            }
            case 10: {
                const uint32_t n = (uint32_t)s.uleb();
                if (n != func_types.size()) refuse("function and code sections disagree");
                for (uint32_t i = 0; i < n; i++) {
                    const uint32_t sz = (uint32_t)s.uleb();
                    if (s.end - s.p < sz) refuse("truncated function body");
                    bodies.push_back({s.p, s.p + sz});
                    s.p += sz;
                }
                break;
            }
            case 11: {
                const uint32_t n = (uint32_t)s.uleb();
                for (uint32_t i = 0; i < n; i++) {
                    if (s.uleb() != 0) refuse("data segment other than an active segment of memory 0");
                    const uint32_t off = (uint32_t)const_expr(s, w->globals, T_I32);
                    const uint32_t k = (uint32_t)s.uleb();
                    if (s.end - s.p < k) refuse("truncated data segment");
                    datas.push_back({off, s.p, k});
                    s.p += k;
                }
                break;
            }
            case 12: refuse("bulk-memory data count section is not supported");
            default: refuse("unknown section " + std::to_string(id));
        }
        if (id != 0 && s.p != s.end) refuse("section " + std::to_string(id) + " has trailing bytes");
    }
    if (bodies.size() != func_types.size()) refuse("function and code sections disagree");
    if (!have_mem) { w->init_pages = 0; w->decl_max_pages = 0; }
    w->table.assign(have_table ? table_min : 0, NO_FUNC);
    for (auto& e : elems) {
        if ((uint64_t)e.first + e.second.size() > w->table.size()) refuse("element segment outside the table");
        std::copy(e.second.begin(), e.second.end(), w->table.begin() + e.first);
    }
    w->image.assign((size_t)w->init_pages * PAGE_WORDS, 0);
    for (auto& d : datas) {
        if ((uint64_t)d.off + d.n > (uint64_t)w->init_pages * 65536) refuse("data segment outside the memory");
        memcpy((uint8_t*)w->image.data() + d.off, data + d.p, d.n);
    }
    for (size_t i = 0; i < bodies.size(); i++) {
        const uint32_t fi = w->nimports + (uint32_t)i;
        translate(w, fi, Reader{data, bodies[i].first, bodies[i].second}, w->types[func_types[i]], w->fns[fi].nparams);
    }
    if (w->code.size() >= EXIT_PC) refuse("module too large");
    if (w->code.empty()) w->code.push_back({I_UNREACHABLE, 0, 0, 0});
    if (w->table.empty()) w->table.push_back(NO_FUNC);
}

void upload(b2g_wasm* w) {
    DevGuard g(w->device);
    CUDA_CHECK(cudaMalloc(&w->d_code, w->code.size() * sizeof(Ins)));
    CUDA_CHECK(cudaMemcpy(w->d_code, w->code.data(), w->code.size() * sizeof(Ins), cudaMemcpyHostToDevice));
    CUDA_CHECK(cudaMalloc(&w->d_fns, std::max<size_t>(1, w->fns.size()) * sizeof(Fn)));
    if (!w->fns.empty()) CUDA_CHECK(cudaMemcpy(w->d_fns, w->fns.data(), w->fns.size() * sizeof(Fn), cudaMemcpyHostToDevice));
    CUDA_CHECK(cudaMalloc(&w->d_table, w->table.size() * 4));
    CUDA_CHECK(cudaMemcpy(w->d_table, w->table.data(), w->table.size() * 4, cudaMemcpyHostToDevice));
    CUDA_CHECK(cudaMalloc(&w->d_image, std::max<size_t>(1, w->image.size()) * 4));
    if (!w->image.empty()) CUDA_CHECK(cudaMemcpy(w->d_image, w->image.data(), w->image.size() * 4, cudaMemcpyHostToDevice));
    std::vector<uint64_t> gi;
    for (auto& x : w->globals) gi.push_back(x.init);
    CUDA_CHECK(cudaMalloc(&w->d_glob, std::max<size_t>(1, gi.size()) * 8));
    if (!gi.empty()) CUDA_CHECK(cudaMemcpy(w->d_glob, gi.data(), gi.size() * 8, cudaMemcpyHostToDevice));
}

template <class T>
struct DevBuf {
    T* p = nullptr;
    explicit DevBuf(size_t n) { CUDA_CHECK(cudaMalloc(&p, std::max<size_t>(n, 1) * sizeof(T))); }
    ~DevBuf() { cudaFree(p); }
    DevBuf(const DevBuf&) = delete;
};

size_t lane_bytes(const b2g_wasm* w, size_t io_bytes) {
    return (size_t)w->lim.max_pages * 65536 + (size_t)w->lim.stack_slots * 8 + (size_t)w->lim.max_depth * 8 + io_bytes + 4;
}

// Runs `count` lanes of mode `mode` in chunks that fit the device-memory budget.  io_in / io_out: per-lane bytes of
// the chunk's inputs (values or run arguments) and outputs; stage(prog, first, n) uploads a chunk's inputs and
// collect(first, n) copies its outputs back.
template <class Stage, class Collect>
void run_lanes(b2g_ctx* ctx, b2g_wasm* w, Prog base, uint32_t count, size_t io_in, size_t io_out, uint32_t* status_out,
               Stage&& stage, Collect&& collect) {
    const CtxView cv = ctx_idle(ctx);
    if (cv.device != w->device) throw_error(B2G_E_SHAPE, "the module was loaded on another device");
    DevGuard g(cv.device);
    cudaStream_t st = cv.st;
    const size_t per = lane_bytes(w, io_in + io_out);
    size_t budget = w->lim.budget_bytes;
    if (!budget) {
        size_t fr = 0, tot = 0;
        CUDA_CHECK(cudaMemGetInfo(&fr, &tot));
        budget = std::min<size_t>(fr / 2, (size_t)32 << 30);
    }
    if (budget / per < 32)
        throw_error(B2G_E_SHAPE, "wasm: the device-memory budget (" + std::to_string(budget) + " B) is below one warp's lane state (32 x " +
                                     std::to_string(per) + " B): raise budget_bytes or lower max_pages / stack_slots / max_depth");
    size_t chunk = budget / per / 32 * 32;
    chunk = std::min<size_t>(chunk, ((size_t)count + 31) / 32 * 32);
    DevBuf<uint32_t> mem(chunk * w->lim.max_pages * (size_t)PAGE_WORDS);
    DevBuf<uint64_t> slots(chunk * (size_t)w->lim.stack_slots);
    DevBuf<uint2> frames(chunk * (size_t)w->lim.max_depth);
    DevBuf<uint8_t> in(chunk * io_in), out(chunk * io_out);
    DevBuf<uint32_t> stat(chunk);
    Prog P = base;
    P.code = w->d_code; P.fns = w->d_fns; P.table = w->d_table; P.table_size = (uint32_t)w->table.size();
    P.global_init = w->d_glob; P.nglobals = (uint32_t)w->globals.size();
    P.image = w->d_image; P.image_words = (uint32_t)w->image.size();
    P.init_pages = w->init_pages; P.max_pages = w->lim.max_pages;
    P.slot_cap = w->lim.stack_slots; P.depth_cap = w->lim.max_depth; P.fuel = w->lim.fuel;
    P.mem = mem.p; P.slots = slots.p; P.frames = frames.p; P.status = stat.p;
    for (uint32_t first = 0; first < count; first += (uint32_t)chunk) {
        const uint32_t n = (uint32_t)std::min<size_t>(chunk, count - first);
        P.lanes = n;
        stage(P, in.p, out.p, first, n, st);
        wasm_kernel<<<(n + 127) / 128, 128, 0, st>>>(P);
        CUDA_CHECK(cudaGetLastError());
        g_launch_count += 1;
        collect(out.p, first, n, st);
        CUDA_CHECK(cudaMemcpyAsync(status_out + first, stat.p, (size_t)n * 4, cudaMemcpyDeviceToHost, st));
        CUDA_CHECK(cudaStreamSynchronize(st));
    }
}

void check_limits(const b2g_wasm* w, const b2g_wasm_limits& l) {
    if (l.max_pages < w->init_pages || l.max_pages > 65536) throw_error(B2G_E_SHAPE, "max_pages must be in [the module's initial pages, 65536]");
    if (l.max_pages > w->decl_max_pages) throw_error(B2G_E_SHAPE, "max_pages is above the module's declared maximum");
    if (l.max_depth < 1 || l.max_depth > (1u << 20)) throw_error(B2G_E_SHAPE, "max_depth must be in [1, 2^20]");
    if (l.stack_slots < w->globals.size() + MIN_SLOTS_ABOVE_GLOBALS || l.stack_slots > (1u << 24))
        throw_error(B2G_E_SHAPE, "stack_slots must be in [globals + " + std::to_string(MIN_SLOTS_ABOVE_GLOBALS) + " = " +
                                     std::to_string(w->globals.size() + MIN_SLOTS_ABOVE_GLOBALS) + ", 2^24]");
    if (l.fuel == 0) throw_error(B2G_E_SHAPE, "fuel must be positive");
}

// The defaults are sized from the module (its pages, its globals) and pass check_limits
void default_limits(b2g_wasm* w) {
    w->lim.max_pages = std::min<uint32_t>(w->decl_max_pages, w->init_pages + 5);
    w->lim.max_depth = 256;
    w->lim.stack_slots = (uint32_t)w->globals.size() + 4096;
    w->lim.fuel = DEFAULT_FUEL;
    w->lim.budget_bytes = 0;
    check_limits(w, w->lim);
}

void probe(b2g_ctx* ctx, b2g_wasm* w) {
    for (int k = 0; k < 10; k++) {
        const int f = w->find_export(PROTOCOL[k]);
        if (f < 0) refuse(std::string("the module does not export the circom 2 function ") + PROTOCOL[k] +
                          (w->find_export("getFrLen") >= 0 ? " (it looks like a circom 1 module)" : ""));
        w->fx[k] = (uint32_t)f;
    }
    static const uint32_t want_params[10] = {1, 2, 3, 0, 1, 1, 0, 0, 0, 0};
    static const bool want_result[10] = {false, false, false, true, false, true, true, true, false, true};
    for (int k = 0; k < 10; k++) {
        const Fn& f = w->fns[w->fx[k]];
        const FuncType& t = w->types[f.type_index];
        bool ok = f.entry != NO_FUNC && t.params.size() == want_params[k] && t.results.size() == (want_result[k] ? 1u : 0u);
        for (uint8_t p : t.params) ok = ok && p == T_I32;
        for (uint8_t p : t.results) ok = ok && p == T_I32;
        if (!ok) refuse(std::string("the export ") + PROTOCOL[k] + " does not have the circom 2 signature");
    }
    Prog P = {};
    P.mode = 0;
    memcpy(P.fx, w->fx, sizeof P.fx);
    uint32_t res[16] = {}, status = 0;
    run_lanes(ctx, w, P, 1, 0, 64, &status,
              [&](Prog& p, uint8_t*, uint8_t* out, uint32_t, uint32_t, cudaStream_t st) {
                  p.out = (uint32_t*)out;
                  CUDA_CHECK(cudaMemsetAsync(out, 0, 64, st));
              },
              [&](uint8_t* out, uint32_t, uint32_t, cudaStream_t st) {
                  CUDA_CHECK(cudaMemcpyAsync(res, out, 64, cudaMemcpyDeviceToHost, st));
              });
    if (status != 0) refuse("the module trapped while reporting its field and sizes (lane status " + std::to_string(status) + ")");
    w->info.version = res[0]; w->info.n32 = res[1]; w->info.witness_size = res[10]; w->info.input_size = res[11];
    if (w->info.n32 != 8) refuse("getFieldNumLen32 returned " + std::to_string(w->info.n32) + ": only 8 (a 254-bit field) is supported");
    if (memcmp(res + 2, R_WORDS, 32) != 0) refuse("the circuit's prime is not the BN254 scalar field modulus r");
    if (w->info.witness_size == 0) refuse("the module reports an empty witness");
}

// b2g_wasm_load (circom: the protocol exports, then the probe lane) and b2g_wasm_load_module
int load(b2g_ctx* ctx, const void* bytes, size_t len, b2g_wasm** out, bool circom) {
    return guarded_clear([&] {
        if (!ctx || !bytes || !out) throw_error(B2G_E_SHAPE, "null pointer");
        *out = nullptr;
        std::unique_ptr<b2g_wasm> w(new b2g_wasm);
        w->device = ctx_view(ctx).device;
        load_module(w.get(), (const uint8_t*)bytes, len);
        default_limits(w.get());
        w->info.mem_pages = w->init_pages;
        upload(w.get());
        if (circom) {
            w->circom = true;
            probe(ctx, w.get());
        }
        *out = w.release();
    });
}
}  // namespace

extern "C" {

int b2g_wasm_load_module(b2g_ctx* ctx, const void* bytes, size_t len, b2g_wasm** out) { return load(ctx, bytes, len, out, false); }

int b2g_wasm_load(b2g_ctx* ctx, const void* bytes, size_t len, b2g_wasm** out) { return load(ctx, bytes, len, out, true); }

int b2g_wasm_free(b2g_wasm* w) {
    return guarded([&] { delete w; });
}

int b2g_wasm_info(b2g_wasm* w, b2g_wasm_summary* out) {
    return guarded([&] {
        if (!w || !out) throw_error(B2G_E_SHAPE, "null pointer");
        *out = w->info;
    });
}

int b2g_wasm_get_limits(b2g_wasm* w, b2g_wasm_limits* out) {
    return guarded([&] {
        if (!w || !out) throw_error(B2G_E_SHAPE, "null pointer");
        *out = w->lim;
    });
}

int b2g_wasm_set_limits(b2g_wasm* w, const b2g_wasm_limits* lim) {
    return guarded([&] {
        if (!w || !lim) throw_error(B2G_E_SHAPE, "null pointer");
        check_limits(w, *lim);
        w->lim = *lim;
    });
}

int b2g_wasm_run(b2g_ctx* ctx, b2g_wasm* w, const char* name, uint32_t count, uint32_t nargs, const uint64_t* args,
                 uint64_t* results, uint32_t* status_out) {
    return guarded_clear([&] {
        if (!ctx || !w || !name || !status_out || (nargs && !args) || (count && !results)) throw_error(B2G_E_SHAPE, "null pointer");
        const int f = w->find_export(name);
        if (f < 0) throw_error(B2G_E_SHAPE, std::string("wasm: the module does not export a function ") + name);
        if (w->fns[f].nparams != nargs) throw_error(B2G_E_SHAPE, std::string("wasm: ") + name + " takes " + std::to_string(w->fns[f].nparams) + " arguments");
        if (nargs > 3) throw_error(B2G_E_SHAPE, "wasm: b2g_wasm_run passes at most 3 arguments");
        if (count == 0) return;
        Prog P = {};
        P.mode = 2; P.run_fn = (uint32_t)f; P.run_nargs = nargs;
        run_lanes(ctx, w, P, count, nargs * 8, 8, status_out,
                  [&](Prog& p, uint8_t* in, uint8_t* out, uint32_t first, uint32_t n, cudaStream_t st) {
                      p.run_args = (const uint64_t*)in; p.run_out = (uint64_t*)out;
                      if (nargs) CUDA_CHECK(cudaMemcpyAsync(in, args + (size_t)first * nargs, (size_t)n * nargs * 8, cudaMemcpyHostToDevice, st));
                      CUDA_CHECK(cudaMemsetAsync(out, 0, (size_t)n * 8, st));
                  },
                  [&](uint8_t* out, uint32_t first, uint32_t n, cudaStream_t st) {
                      CUDA_CHECK(cudaMemcpyAsync(results + first, out, (size_t)n * 8, cudaMemcpyDeviceToHost, st));
                  });
    });
}

int b2g_witness_calculate(b2g_ctx* ctx, b2g_wasm* w, uint32_t count, uint32_t n_inputs, const uint64_t* hashes,
                          const uint32_t* counts, const void* values_canon, int sanity_check, void* w_mont_out,
                          uint32_t* status_out) {
    return guarded_clear([&] {
        if (!ctx || !w || (n_inputs && (!hashes || !counts)) || (count && (!w_mont_out || !status_out))) throw_error(B2G_E_SHAPE, "null pointer");
        if (!w->circom) throw_error(B2G_E_SHAPE, "wasm: the module was not loaded as a circom 2 witness calculator (b2g_wasm_load)");
        uint64_t n_values = 0;
        for (uint32_t k = 0; k < n_inputs; k++)
            if ((n_values += counts[k]) > (1u << 24)) throw_error(B2G_E_SHAPE, "too many input values");
        std::vector<uint3> meta;
        meta.reserve(n_values);
        for (uint32_t k = 0; k < n_inputs; k++)
            for (uint32_t i = 0; i < counts[k]; i++) meta.push_back(make_uint3((uint32_t)(hashes[k] >> 32), (uint32_t)hashes[k], i));
        const uint32_t nv = (uint32_t)meta.size();
        if (count == 0) return;
        if (nv && !values_canon) throw_error(B2G_E_SHAPE, "null pointer");
        const uint32_t* vals = (const uint32_t*)values_canon;
        for (size_t e = 0; e < (size_t)count * nv; e++) {
            const uint32_t* x = vals + 8 * e;
            for (int j = 7; j >= 0; j--) {
                if (x[j] != R_WORDS[j]) { if (x[j] > R_WORDS[j]) throw_error(B2G_E_INPUT, "values_canon[" + std::to_string(e) + "] is not below r"); break; }
                if (j == 0) throw_error(B2G_E_INPUT, "values_canon[" + std::to_string(e) + "] is not below r");
            }
        }
        const uint32_t nw = w->info.witness_size;
        if ((uint64_t)(2 + 9ull * nv + 9ull * nw) >= 0xffffffffull) throw_error(B2G_E_SHAPE, "too many calls per witness");
        DevBuf<uint3> d_meta(nv);
        if (nv) CUDA_CHECK(cudaMemcpy(d_meta.p, meta.data(), nv * sizeof(uint3), cudaMemcpyHostToDevice));
        Prog P = {};
        P.mode = 1;
        memcpy(P.fx, w->fx, sizeof P.fx);
        P.value_meta = d_meta.p; P.n_values = nv; P.n_wit = nw; P.sanity = sanity_check ? 1 : 0;
        const size_t in_b = (size_t)nv * 32, out_b = (size_t)nw * 32;
        uint8_t* dst = (uint8_t*)w_mont_out;
        run_lanes(ctx, w, P, count, in_b, out_b, status_out,
                  [&](Prog& p, uint8_t* in, uint8_t* out, uint32_t first, uint32_t n, cudaStream_t st) {
                      p.values = (const uint32_t*)in; p.out = (uint32_t*)out;
                      if (in_b) CUDA_CHECK(cudaMemcpyAsync(in, (const uint8_t*)values_canon + first * in_b, n * in_b, cudaMemcpyHostToDevice, st));
                      CUDA_CHECK(cudaMemsetAsync(out, 0, n * out_b, st));
                  },
                  [&](uint8_t* out, uint32_t first, uint32_t n, cudaStream_t st) {
                      const size_t ne = (size_t)n * nw;
                      wasm_to_mont_kernel<<<(unsigned)((ne + 255) / 256), 256, 0, st>>>((uint32_t*)out, ne);
                      CUDA_CHECK(cudaGetLastError());
                      g_launch_count += 1;
                      CUDA_CHECK(cudaMemcpyAsync(dst + first * out_b, out, n * out_b, cudaMemcpyDeviceToHost, st));
                  });
        // the witness of a lane that did not finish is all zeros
        for (uint32_t i = 0; i < count; i++)
            if (status_out[i]) memset(dst + i * out_b, 0, out_b);
    });
}

}  // extern "C"
