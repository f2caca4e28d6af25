/* Embeds the sm_90a device module (coast_kernels.cubin) into libcoast_rt.so. */
    .section .rodata
    .balign 64
    .global coast_kernels_cubin
    .type coast_kernels_cubin, @object
coast_kernels_cubin:
    .incbin "coast_kernels.cubin"
    .global coast_kernels_cubin_end
coast_kernels_cubin_end:
    .byte 0
    .size coast_kernels_cubin, . - coast_kernels_cubin
    .section .note.GNU-stack,"",@progbits
