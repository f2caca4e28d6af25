/*
 * COAST.h -- the in-code directive surface of COAST, as honoured by the GPU runtime.
 *
 * Same 17 macro names, same spelling of every annotation string as byuccl/coast
 * tests/COAST.h:11-67 (strings must match projects/dataflowProtection/dataflowProtection.h:69-79),
 * so sources written against the reference compile unchanged.
 *
 * Two back ends:
 *   - clang feeding the LLVM pass (define COAST_LLVM_PASS): the macros expand to
 *     __attribute__((annotate("..."))) exactly as the reference expects;
 *   - everything else (gcc / nvcc host code linked against libcoast_rt.so -- the default):
 *     protection is applied at RUN TIME by the launch ABI (include/coast_rt.h), there is no
 *     IR to annotate, and gcc rejects attributes in some positions the tests use them
 *     (`int checkGolden() __NO_xMR {`, tests/matrixMultiply/matrixMultiply.c:115), so in the COMPILED
 *     translation unit the scope directives expand to nothing -- but they are not ignored: the BOARD=b200 pass
 *     preprocesses every source a second time with COAST_SCOPE_SCAN (third back end below), reads the directives
 *     with include/makefiles/coast_scope.c and decides from them which calls become protected launches:
 *       - a function in the SoR (explicit __xMR, or default scope without __DEFAULT_NO_xMR / __NO_xMR) that has a
 *         runtime kernel (include/makefiles/coast_entries.tab) is offloaded;
 *       - __NO_xMR on such a function keeps its calls on the CPU, unprotected, as in the reference;
 *       - an explicit __xMR on a function with no kernel that calls none FAILS THE BUILD, naming it.
 *     What the directives MEAN for the runtime:
 *
 *   directive                        reference meaning (interface.cpp:364-601)          GPU runtime
 *   -------------------------------  -------------------------------------------------  ---------------------------------
 *   __xMR / __NO_xMR                 put fn/global/local in / out of the SoR            SoR = the offloaded kernel body
 *   __DEFAULT_xMR / __DEFAULT_NO_xMR default scope; both DECLARE an int (:20-21)        same declaration is emitted
 *   __xMR_FN_CALL / __SKIP_FN_CALL   replicate / call-once for a callee                 n/a inside a kernel (no calls out)
 *   __xMR_RET_VAL                    replicate the return value                         kernels vote every output element
 *   __xMR_PROT_LIB, __ISR_FUNC       keep signature / never clone                       n/a
 *   __xMR_ALL_AFTER_CALL etc.        clone args after call (scanf-style)                n/a
 *   __COAST_VOLATILE, __COAST_NO_INLINE  plain GCC attributes                           identical
 *   *_WRAPPER_REGISTER / _CALL       name-mangling helpers                              identical token pasting
 */
#ifndef __COAST_MACROS__
#define __COAST_MACROS__

#if defined(COAST_LLVM_PASS)
#  define COAST_ANNOTATE_(s) __attribute__((annotate(s)))
#elif defined(COAST_SCOPE_SCAN)
/* `gcc -E` only: the directive survives preprocessing as a token sequence that include/makefiles/coast_scope.c reads to
 * decide the sphere of replication (what processAnnotations() does with llvm.global.annotations, interface.cpp:364-532) */
#  define COAST_ANNOTATE_(s) __coast_anno__(s)
#else
#  define COAST_ANNOTATE_(s)
#endif

/* scope of replication: variables and functions */
#define __xMR     COAST_ANNOTATE_("xMR")
#define __NO_xMR  COAST_ANNOTATE_("no_xMR")

/* per-callee behaviour (-replicateFnCalls / -skipLibCalls equivalents) */
#define __xMR_FN_CALL   COAST_ANNOTATE_("xMR_call")
#define __SKIP_FN_CALL  COAST_ANNOTATE_("coast_call_once")

/* default scope for the translation unit; the declared int is part of the contract */
#define __DEFAULT_xMR     int COAST_ANNOTATE_("set_xMR_default") __xMR_DEFAULT_BEHAVIOR__;
#define __DEFAULT_NO_xMR  int COAST_ANNOTATE_("set_no_xMR_default") __xMR_DEFAULT_BEHAVIOR__;

/* plain compiler attributes */
#define __COAST_VOLATILE   __attribute__((used))
#define __COAST_NO_INLINE  __attribute__((noinline))

/* function kinds */
#define __ISR_FUNC      COAST_ANNOTATE_("isr_function")
#define __xMR_RET_VAL   COAST_ANNOTATE_("repl_return_val")
#define __xMR_PROT_LIB  COAST_ANNOTATE_("protected_lib")

/* clone-after-call: every argument, or the listed ones (name, 1_2_3) */
#define __xMR_ALL_AFTER_CALL         COAST_ANNOTATE_("clone-after-call-")
#define __xMR_AFTER_CALL(fname, x)   fname##_CLONE_AFTER_CALL_##x

/* wrappers the pass recognises by suffix */
#define MALLOC_WRAPPER_REGISTER(fname)        void* fname##_COAST_WRAPPER(size_t size)
#define MALLOC_WRAPPER_CALL(fname, x)         fname##_COAST_WRAPPER((x))
#define PRINTF_WRAPPER_REGISTER(fname)        int fname##_COAST_WRAPPER(const char* format, ...)
#define PRINTF_WRAPPER_CALL(fname, fmt, ...)  fname##_COAST_WRAPPER(fmt, __VA_ARGS__)
#define GENERIC_COAST_WRAPPER(fname)          fname##_COAST_WRAPPER

/* verification overrides */
#define __COAST_IGNORE_GLOBAL(name)  COAST_ANNOTATE_("no-verify-" #name)
#define __NO_xMR_ARG(num)            COAST_ANNOTATE_("no_xMR_arg-" #num)

#endif /* __COAST_MACROS__ */
