// bin_b200 -- wgmma.mma_async wrappers for sm_90a: D(64 x N, fp32, registers) (+)= A(64 x 16, fp16, smem) * B(16 x N, fp16,
// smem).  The instruction's operand list has to be spelled out per N, hence one specialisation per supported N
// (BIN_R*: accumulator placeholders, BIN_D8: their constraints).  TA / TB = 1 selects an MN-major (transposed) operand.
#pragma once
#include <stdint.h>

namespace binb {

template <int N, int TA = 0, int TB = 0>
struct Wgmma;

#define BIN_R0 "%0,%1,%2,%3,%4,%5,%6,%7"
#define BIN_R1 "%8,%9,%10,%11,%12,%13,%14,%15"
#define BIN_R2 "%16,%17,%18,%19,%20,%21,%22,%23"
#define BIN_R3 "%24,%25,%26,%27,%28,%29,%30,%31"
#define BIN_R4 "%32,%33,%34,%35,%36,%37,%38,%39"
#define BIN_R5 "%40,%41,%42,%43,%44,%45,%46,%47"
#define BIN_R6 "%48,%49,%50,%51,%52,%53,%54,%55"
#define BIN_R7 "%56,%57,%58,%59,%60,%61,%62,%63"
#define BIN_R8 "%64,%65,%66,%67,%68,%69,%70,%71"
#define BIN_R9 "%72,%73,%74,%75,%76,%77,%78,%79"
#define BIN_R10 "%80,%81,%82,%83,%84,%85,%86,%87"
#define BIN_R11 "%88,%89,%90,%91,%92,%93,%94,%95"
#define BIN_R12 "%96,%97,%98,%99,%100,%101,%102,%103"
#define BIN_R13 "%104,%105,%106,%107,%108,%109,%110,%111"
#define BIN_R14 "%112,%113,%114,%115,%116,%117,%118,%119"
#define BIN_R15 "%120,%121,%122,%123,%124,%125,%126,%127"
#define BIN_D8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
#define BIN_WGMMA(N, REGS, TAIL, ...)                                                                                     \
  template <int TA, int TB>                                                                                          \
  struct Wgmma<N, TA, TB> {                                                                                          \
    static __device__ __forceinline__ void mma(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t scale_d) {      \
      asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" TAIL ";\n\t}"                                             \
                   : __VA_ARGS__                                                                                     \
                   : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));                                              \
    }                                                                                                                \
  };
BIN_WGMMA(16, , "10, 0;\n\twgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {" BIN_R0 "}, %8, %9, p, 1, 1, %11, %12", BIN_D8(0))
BIN_WGMMA(32, , "18, 0;\n\twgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {" BIN_R0 "," BIN_R1 "}, %16, %17, p, 1, 1, %19, %20", BIN_D8(0), BIN_D8(8))
BIN_WGMMA(48, , "26, 0;\n\twgmma.mma_async.sync.aligned.m64n48k16.f32.f16.f16 {" BIN_R0 "," BIN_R1 "," BIN_R2 "}, %24, %25, p, 1, 1, %27, %28", BIN_D8(0), BIN_D8(8), BIN_D8(16))
BIN_WGMMA(64, , "34, 0;\n\twgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {" BIN_R0 "," BIN_R1 "," BIN_R2 "," BIN_R3 "}, %32, %33, p, 1, 1, %35, %36", BIN_D8(0), BIN_D8(8), BIN_D8(16), BIN_D8(24))
BIN_WGMMA(96, , "50, 0;\n\twgmma.mma_async.sync.aligned.m64n96k16.f32.f16.f16 {" BIN_R0 "," BIN_R1 "," BIN_R2 "," BIN_R3 "," BIN_R4 "," BIN_R5 "}, %48, %49, p, 1, 1, %51, %52", BIN_D8(0), BIN_D8(8), BIN_D8(16), BIN_D8(24), BIN_D8(32), BIN_D8(40))
BIN_WGMMA(128, , "66, 0;\n\twgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {" BIN_R0 "," BIN_R1 "," BIN_R2 "," BIN_R3 "," BIN_R4 "," BIN_R5 "," BIN_R6 "," BIN_R7 "}, %64, %65, p, 1, 1, %67, %68", BIN_D8(0), BIN_D8(8), BIN_D8(16), BIN_D8(24), BIN_D8(32), BIN_D8(40), BIN_D8(48), BIN_D8(56))
BIN_WGMMA(256, , "130, 0;\n\twgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 {" BIN_R0 "," BIN_R1 "," BIN_R2 "," BIN_R3 "," BIN_R4 "," BIN_R5 "," BIN_R6 "," BIN_R7 "," BIN_R8 "," BIN_R9 "," BIN_R10 "," BIN_R11 "," BIN_R12 "," BIN_R13 "," BIN_R14 "," BIN_R15 "}, %128, %129, p, 1, 1, %131, %132", BIN_D8(0), BIN_D8(8), BIN_D8(16), BIN_D8(24), BIN_D8(32), BIN_D8(40), BIN_D8(48), BIN_D8(56), BIN_D8(64), BIN_D8(72), BIN_D8(80), BIN_D8(88), BIN_D8(96), BIN_D8(104), BIN_D8(112), BIN_D8(120))
#undef BIN_WGMMA
#undef BIN_D8
#undef BIN_R0
#undef BIN_R1
#undef BIN_R2
#undef BIN_R3
#undef BIN_R4
#undef BIN_R5
#undef BIN_R6
#undef BIN_R7
#undef BIN_R8
#undef BIN_R9
#undef BIN_R10
#undef BIN_R11
#undef BIN_R12
#undef BIN_R13
#undef BIN_R14
#undef BIN_R15

}  // namespace binb
